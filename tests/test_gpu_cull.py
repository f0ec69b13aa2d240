"""Exact culling on needle splats far from their tiles (DESIGN.md section 4): the binning-time tile mask (tile_keep_mask on the API
path, warp_tile_keep_mask on the fused path) and the blend kernels' sub-tile culls may drop only (pixel, Gaussian) pairs the reference
itself skips.

Scenes are screen-space needles (sigma_major 200-2000 px, 60-180 px at the corners; sigma_minor <= 0.3 px) whose centres lie hundreds
of pixels outside small images, strips one or two tiles tall and the corners of a 1080p frame, where a rectangle of at most 64 tiles can
lie far from the centre and q = hA dx^2 + hC dy^2 + B dx dy cancels large terms; in-image needles and rectangles of more than 64 tiles
(kept whole by the tile mask) are the controls, and stress the blend kernels' sub-tile culls instead.  Each Gaussian's opacity puts the reference's best pixel in one of its tiles at
alpha (1 + eps) / 255.
  - decision audit: every instance the tile mask drops (the lists with culling off minus the lists with culling on) is checked against
    the reference's pinned pair_power over the tile's pixel centres (tests/native/math_host.cpp), on the API and fused paths and in
    every binning mode;
  - outputs with culling on (the product default) against the reference's kernels, bit for bit, and significance counts against the
    oracle's exact counts on its own lists;
  - gradients against the oracle's backward run on its own lists (an instance we wrongly drop is visible there);
  - a 65552 x 32 strip (4097 tiles wide): the fused path's warp-cooperative mask must equal the API path's per-lane mask."""
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lightgaussian_b200 import capi
from lightgaussian_b200.synth import camera_from_pose
from oracle.lgo import Oracle
from tests import util
from tests.test_host_math import lib  # noqa: F401  (the host build of lgr_math.cuh, built on demand)
from tests.util import oracle_from_geometry, read_state, run_ours, run_ref, view_from_camera

pytestmark = pytest.mark.gpu

needs_ref = pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref/libref_rasterizer.so not built (needs the reference checkout)")

FOV = math.radians(60.0)
DEG = 1
EPS = (1e-3, 5e-3, 2e-2)
GRAD_TOL = 1e-3

# name -> W, H, kind, centre distance range (px), number of candidate needles, minimum at-threshold tiles the audit must see
FAMILIES = {
    "strip_1024x16": (1024, 16, "far", (300.0, 1200.0), 1500, 1000),
    "strip_16x1024": (16, 1024, "far", (300.0, 1200.0), 1500, 1000),
    "strip_2048x32": (2048, 32, "far", (300.0, 1200.0), 1500, 300),
    "small_128x128": (128, 128, "far", (300.0, 1500.0), 1500, 500),
    "small_96x64": (96, 64, "far", (300.0, 1500.0), 1500, 300),
    "corner_1080p": (1920, 1080, "corner", None, 1500, 300),
    "in_image_256": (256, 256, "inside", (0.0, 100.0), 1500, 500),
}


def _candidates(W, H, kind, drange, n, rng):
    """screen-space needles: centre (px), direction theta of the major axis, sigma_major / minor (px)"""
    d = rng.uniform(*drange, n) if drange else None
    diag = rng.random(n) < 0.25                            # 45 degrees (and 135) with integer centres
    if kind == "corner":
        # the centre beyond a corner by (Dx, Dy) with 3 sigma_major - Dx, 3 sigma_major - Dy <= 128 px, so that the clamped rectangle is
        # at most 8 x 8 tiles, and the needle's axis through a target pixel near the corner (diagonal: on the 45 degree line).  A pixel
        # there keeps G = exp(-d^2 / 2 sigma^2) > 1/255 only for sigma_major below ~200 px.
        sM = rng.uniform(60.0, 180.0, n)
        lo, hi = 0.7 * sM, np.minimum(128.0, sM)
        Dx, Dy = 3 * sM - rng.uniform(lo, hi), 3 * sM - rng.uniform(lo, hi)
        Dy[diag] = Dx[diag] = np.round(Dx[diag])
        a, b = rng.uniform(0, 0.3, n) * (3 * sM - Dx), rng.uniform(0, 0.3, n) * (3 * sM - Dy)
        b[diag] = a[diag]
        right, below = rng.integers(0, 2, n), rng.integers(0, 2, n)
        sx, sy = np.where(right == 1, 1.0, -1.0), np.where(below == 1, 1.0, -1.0)
        cx0, cy0 = np.where(right == 1, W - 1, 0), np.where(below == 1, H - 1, 0)
        tx, ty = cx0 - sx * a, cy0 - sy * b
        px, py = cx0 + sx * Dx, cy0 + sy * Dy
        d = np.hypot(px - tx, py - ty)
        phi = np.arctan2(py - ty, px - tx)
    else:
        tx, ty = rng.uniform(0, W - 1, n), rng.uniform(0, H - 1, n)
        phi = np.where(diag, np.pi / 4 + np.pi / 2 * rng.integers(0, 4, n), rng.uniform(0.0, 2 * np.pi, n))
        perp = rng.uniform(-1.0, 1.0, n)
        px = tx + d * np.cos(phi) - perp * np.sin(phi)
        py = ty + d * np.sin(phi) + perp * np.cos(phi)
        px[diag], py[diag] = np.round(px[diag]), np.round(py[diag])
    # phi: direction from the target point to the centre, along the major axis (theta)
    theta = np.mod(phi, np.pi)
    if kind == "inside":
        sM = rng.uniform(20.0, 200.0, n)
    elif kind == "far":
        sM = np.clip(d / rng.uniform(0.5, 3.2, n), 200.0, 2000.0)
    sm = rng.uniform(0.05, 0.3, n)
    keep = np.ones(n, bool)
    if kind in ("far", "corner"):
        ox = np.maximum(np.maximum(-px, px - (W - 1)), 0.0)
        oy = np.maximum(np.maximum(-py, py - (H - 1)), 0.0)
        keep = np.hypot(ox, oy) >= (drange[0] if kind == "far" else 0.0)
    return px[keep], py[keep], theta[keep], sM[keep], sm[keep]


def _leaves(W, H, px, py, theta, sM, sm, rng):
    """GaussianModel leaves of needles at depth ~4 seen by an identity-pose camera (x right, y down, z forward)"""
    n = px.size
    fx = W / (2.0 * math.tan(FOV / 2))
    z = 4.0 + 1e-3 * rng.permutation(n)
    xyz = np.stack([(px - (W - 1) / 2) * z / fx, (py - (H - 1) / 2) * z / fx, z], 1)
    scaling = np.log(np.stack([sM * z / fx, sm * z / fx, sm * z / fx], 1))
    rotation = np.stack([np.cos(theta / 2), np.zeros(n), np.zeros(n), np.sin(theta / 2)], 1)
    M = (DEG + 1) ** 2
    f32 = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    return dict(xyz=f32(xyz), features_dc=f32(rng.standard_normal((n, 1, 3))), features_rest=f32(0.2 * rng.standard_normal((n, M - 1, 3))),
                scaling=f32(scaling), rotation=f32(rotation), opacity=np.zeros((n, 1), np.float32))


def _activated(raw):
    """the activated inputs exactly as torch computes them on the GPU (the fused kernels reproduce these bit for bit)"""
    t = {k: torch.from_numpy(v).cuda() for k, v in raw.items()}
    with torch.no_grad():
        act = dict(means3D=t["xyz"], scales=torch.exp(t["scaling"]), rotations=F.normalize(t["rotation"]), opacities=torch.sigmoid(t["opacity"]),
                   shs=torch.cat((t["features_dc"], t["features_rest"]), dim=1))
    return {k: np.ascontiguousarray(v.cpu().numpy()) for k, v in act.items()}


def _p(a):
    import ctypes as C
    return a.ctypes.data_as(C.c_void_p)


def _tile_max_power(lib, view, geom, tile, gid):
    """the reference's largest blending power (pinned pair_power, power <= 0) over the pixel centres of tile `tile` for Gaussian `gid`"""
    gx = (view.W + 15) // 16
    tx, ty = tile % gx, tile // gx
    f32 = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    i32 = lambda a: np.ascontiguousarray(a, np.int32)  # noqa: E731
    m2, co = geom["means2D"][gid], geom["conic_opacity"][gid]
    x0, y0 = i32(16 * tx), i32(16 * ty)
    x1, y1 = i32(np.minimum(16 * tx + 15, view.W - 1)), i32(np.minimum(16 * ty + 15, view.H - 1))
    out = np.empty(tile.size, np.float32)
    lib.mh_rect_max_power(int(tile.size), _p(f32(m2[:, 0])), _p(f32(m2[:, 1])), _p(f32(co[:, 0])), _p(f32(co[:, 1])), _p(f32(co[:, 2])),
                          _p(x0), _p(x1), _p(y0), _p(y1), _p(out))
    return out.astype(np.float64)


def _instances(st):
    """(tile, Gaussian) pairs of a forward state's per-tile lists, in list order"""
    r = st["ranges"].astype(np.int64)
    tile = np.repeat(np.arange(r.shape[0]), r[:, 1] - r[:, 0])
    gid = np.concatenate([st["point_list"][a:b] for a, b in r]) if tile.size else np.zeros(0, np.uint32)
    return tile, gid.astype(np.int64)


def _last_contributor(view, st):
    """per pixel, the Gaussian at which its blend stopped (n_contrib counts list entries, so it shrinks with the culled lists; the
    Gaussian it points at must not change), -1 where none contributed"""
    gx = (view.W + 15) // 16
    y, x = np.divmod(np.arange(view.W * view.H), view.W)
    start = st["ranges"][(y // 16) * gx + x // 16, 0].astype(np.int64)
    n = st["n_contrib"].astype(np.int64)
    pl = np.append(st["point_list"].astype(np.int64), -1)
    return np.where(n > 0, pl[np.where(n > 0, start + n - 1, -1)], -1)


def _rect_tiles(view, geom):
    """every (tile, Gaussian) pair of the reference's rectangles, from the oracle's own binning"""
    pl, ranges = Oracle().bin(view, geom["means2D"], geom["depths"], geom["radii"], geom["tiles_touched"])
    return _instances(dict(ranges=ranges, point_list=pl))


class Scene:
    def __init__(self, name, lib, seed=0):
        W, H, kind, drange, n, self.min_at = FAMILIES[name]
        rng = np.random.default_rng(zlib.crc32(name.encode()) + seed)
        cam = camera_from_pose(np.eye(3), np.zeros(3), W, H, FOV)
        self.view = view_from_camera(cam, (0.0, 0.0, 0.0), DEG, 1.0)
        c = _candidates(W, H, kind, drange, n, rng)
        raw = _leaves(W, H, *c, rng)
        o = Oracle()
        act = _activated(raw)
        g = o.preprocess(self.view, act["means3D"], act["opacities"], shs=act["shs"], scales=act["scales"], rotations=act["rotations"])
        if kind == "corner":           # off-screen centres whose clamped rectangle is at most 8 x 8 tiles
            r = g["radii"].astype(np.float64)
            m = g["means2D"].astype(np.float64)
            w = np.clip(np.floor((m[:, 0] + r + 15) / 16), 0, (W + 15) // 16) - np.clip(np.floor((m[:, 0] - r) / 16), 0, (W + 15) // 16)
            h = np.clip(np.floor((m[:, 1] + r + 15) / 16), 0, (H + 15) // 16) - np.clip(np.floor((m[:, 1] - r) / 16), 0, (H + 15) // 16)
            sel = (g["radii"] > 0) & (w <= 8) & (h <= 8)
            raw = {k: np.ascontiguousarray(v[sel]) for k, v in raw.items()}
            act = {k: np.ascontiguousarray(v[sel]) for k, v in act.items()}
            g = {k: np.ascontiguousarray(v[sel]) for k, v in g.items()}
        self.P = raw["xyz"].shape[0]
        # opacity: one target tile per Gaussian whose best pixel has 1e-3 < G < 0.9 gets alpha (1 + eps) / 255 there
        tile, gid = _rect_tiles(self.view, g)
        G = np.exp(_tile_max_power(lib, self.view, g, tile, gid))
        ok = (G > 1e-3) & (G < 0.9) & (G > (1.0 + max(EPS)) / 255.0)
        pick = np.full(self.P, -1)
        order = rng.permutation(tile.size)
        pick[gid[order][ok[order]]] = order[ok[order]]
        eps = rng.choice(EPS, self.P)
        G_pick = np.where(pick >= 0, G[np.maximum(pick, 0)], 1.0)
        o_act = np.where(pick >= 0, (1.0 + eps) / (255.0 * G_pick), rng.uniform(0.05, 1.0, self.P))
        raw["opacity"] = np.log(o_act / (1.0 - o_act)).astype(np.float32).reshape(-1, 1)
        self.raw = raw
        self.act = _activated(raw)         # the activated opacity bits the kernels see
        self.targets = int((pick >= 0).sum())


_scenes = {}


def scene(name, lib):
    if name not in _scenes:
        _scenes[name] = Scene(name, lib)
    return _scenes[name]


def _settings(view):
    from lightgaussian_b200.rasterizer import GaussianRasterizationSettings
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    return GaussianRasterizationSettings(view.H, view.W, view.tanfovx, view.tanfovy, t(view.bg), view.scale_modifier, t(view.viewmatrix),
                                         t(view.projmatrix), view.sh_degree, t(view.campos), False, False, False)


def run_fused(view, raw, tile_cull=True, bin_mode=None):
    """the fused forward (lgr_forward_raw) of GaussianModel leaves, with the state its backward reads"""
    from lightgaussian_b200.rasterizer import _forward_raw_native
    leaves = [torch.from_numpy(raw[k]).cuda() for k in util.LEAVES]
    capi.set_tile_culling(tile_cull)
    capi.set_binning_mode(capi.DEFAULT_BINNING_MODE if bin_mode is None else bin_mode)
    try:
        with torch.no_grad():
            _, _, R, color, radii, geom, binning, img, _ = _forward_raw_native(False, _settings(view), *leaves)
        torch.cuda.synchronize()
        st = read_state(view, leaves[0].shape[0], R, radii.cpu().numpy(), geom, binning, img)
    finally:
        capi.set_tile_culling(True)
        capi.set_binning_mode(capi.DEFAULT_BINNING_MODE)
    st.update(color=color.cpu().numpy(), num_rendered=R)
    return st


def _assert_same_lists(a, b, what):
    np.testing.assert_array_equal(a["ranges"], b["ranges"], err_msg=f"{what}: ranges")
    np.testing.assert_array_equal(a["point_list"], b["point_list"], err_msg=f"{what}: point_list")


def _audit(lib, view, geom, full, cull):
    """(dropped instances at which the reference blends a pixel, at-threshold instances checked, instances dropped)"""
    ft, fg = _instances(full)
    ct, cg = _instances(cull)
    P = geom["radii"].shape[0]
    kept = np.isin(ft * P + fg, ct * P + cg)
    assert kept.sum() == ct.size, "the culled lists hold instances the unculled lists do not"
    for t in range(full["ranges"].shape[0]):            # the culled list of a tile is an order-preserving subsequence
        a = full["point_list"][full["ranges"][t, 0]:full["ranges"][t, 1]]
        b = cull["point_list"][cull["ranges"][t, 0]:cull["ranges"][t, 1]]
        if b.size:
            np.testing.assert_array_equal(a[np.isin(a, b)], b, err_msg=f"tile {t}")
    o = geom["conic_opacity"][fg, 3].astype(np.float64)
    alpha = o * np.exp(_tile_max_power(lib, view, geom, ft, fg))
    blends = alpha >= (1.0 / 255.0) * (1.0 - 1e-6)
    at = blends & (alpha < 1.03 / 255.0)
    return int((blends & ~kept).sum()), int(at.sum()), int((~kept).sum())


@pytest.mark.parametrize("bin_mode", [0, 1, 2])
@pytest.mark.parametrize("name", list(FAMILIES))
def test_tile_mask_drops_only_pairs_the_reference_skips(lib, name, bin_mode):
    s = scene(name, lib)
    assert s.targets > 0.5 * s.P, f"{s.targets} of {s.P} needles have a target tile"
    v = s.view
    api = {c: run_ours(v, s.act, tile_cull=c, bin_mode=bin_mode) for c in (False, True)}
    fused = {c: run_fused(v, s.raw, tile_cull=c, bin_mode=bin_mode) for c in (False, True)}
    g = fused[True]["geom"]
    vis = g["radii"] > 0
    np.testing.assert_array_equal(g["conic_opacity"][vis, 3], s.act["opacities"].reshape(-1)[vis])
    for path, runs in (("API", api), ("fused", fused)):
        bad, at, dropped = _audit(lib, v, g, runs[False], runs[True])
        print(f"{name} binning mode {bin_mode} {path}: {dropped} instances dropped, {at} at the threshold, {bad} wrongly")
        assert at >= s.min_at, f"only {at} at-threshold instances (want {s.min_at})"
        assert bad == 0, f"{name}, {path} path: the tile mask dropped {bad} instances in which the reference blends a pixel ({at} at the threshold)"
        if name != "in_image_256":
            assert dropped > 0
    for c in (False, True):
        _assert_same_lists(api[c], fused[c], f"API vs fused, tile culling {c}")
        np.testing.assert_array_equal(api[c]["color"], fused[c]["color"])
    for k in ("color", "final_T", "radii"):
        np.testing.assert_array_equal(api[True][k], api[False][k], err_msg=k)
    np.testing.assert_array_equal(_last_contributor(v, api[True]), _last_contributor(v, api[False]))


@needs_ref
@pytest.mark.parametrize("name", list(FAMILIES))
def test_outputs_equal_the_reference_kernels(lib, name):
    """culling on (the product default): image, radii and final_T bit-identical to the reference's kernels in both blend modes and in
    deterministic mode, the fused render too, every pixel's blend stopping at the same Gaussian; significance counts equal the oracle's
    exact counts on its own lists"""
    s = scene(name, lib)
    v = s.view
    ref = run_ref(v, s.act)
    runs = {"blend0": run_ours(v, s.act), "blend1": run_ours(v, s.act, blend_mode=1), "fused": run_fused(v, s.raw)}
    capi.set_deterministic(True)
    try:
        runs["deterministic"] = run_ours(v, s.act)
        runs["fused_deterministic"] = run_fused(v, s.raw)
    finally:
        capi.set_deterministic(False)
    for tag, ours in runs.items():
        for k in ("color", "radii", "final_T"):
            np.testing.assert_array_equal(ours[k], ref[k], err_msg=f"{tag}: {k}")
        np.testing.assert_array_equal(_last_contributor(v, ours), _last_contributor(v, ref), err_msg=f"{tag}: last contributor")
    for blend_mode in (0, 1):
        ours = run_ours(v, s.act, count=True, blend_mode=blend_mode)
        exact = oracle_from_geometry(Oracle(), v, ours["geom"], count=True)
        np.testing.assert_array_equal(ours["color"], ref["color"])
        if not exact["fragile"].any():
            np.testing.assert_array_equal(ours["gaussians_count"], exact["gaussians_count"])
        else:
            assert np.abs(ours["gaussians_count"].astype(np.int64) - exact["gaussians_count"]).sum() <= 64 * int(exact["fragile"].sum())


@pytest.mark.parametrize("name", list(FAMILIES))
def test_gradients_equal_the_oracle_on_its_own_lists(lib, name):
    """the backward of the culled forward against the oracle's backward on its own (unculled) lists and forward state, in float32: a far
    needle's power cancels terms of 1e5-1e7, so a float64 evaluation of it differs from the reference's float32 one by several percent
    of alpha and is no arbiter here; the oracle keeps the reference's float32 operation order.  The blend backward's own outputs (the
    per-Gaussian sums over the pairs a list holds, where a wrongly dropped instance shows), norm-wise: a needle's screen-space mean
    gradient sums A dx + B dy, which cancels along the axis, so single small entries carry no correct digit in any float32 evaluation
    order, and the preprocess backward multiplies that noise by the needles' large Jacobian terms"""
    s = scene(name, lib)
    v = s.view
    dpix = np.random.default_rng(5).standard_normal((3, v.H, v.W)).astype(np.float32)
    ours = run_ours(v, s.act, dL_dpix=dpix)
    geom = ours["geom"]
    o = Oracle()
    f = oracle_from_geometry(o, v, geom, want_fragile=False)
    g2 = o.blend_backward(v, s.P, f["ranges"], f["point_list"], geom["means2D"], geom["conic_opacity"], geom["rgb"], f["final_T"],
                          f["n_contrib"], dpix)
    mine = ours["grads"]
    checks = {"dL_dmeans2D": (mine["dL_dmeans2D"][:, :2], g2["dL_dmean2D"]), "dL_dcolors": (mine["dL_dcolors"], g2["dL_dcolor"]),
              "dL_dopacity": (mine["dL_dopacity"].reshape(-1), g2["dL_dopacity"])}
    for k, (a, b) in checks.items():
        b = np.asarray(b).reshape(a.shape)
        assert np.isfinite(a).all(), k
        assert util.rel_inf(a, b) <= GRAD_TOL, f"{name} {k}: rel_inf {util.rel_inf(a, b)}"
        assert util.rel_l2(a, b) <= GRAD_TOL, f"{name} {k}: rel_l2 {util.rel_l2(a, b)}"
    if util.have_ref():
        ref = run_ref(v, s.act, dL_dpix=dpix)["grads"]
        for k in ("dL_dmeans2D", "dL_dcolors", "dL_dopacity"):
            a, b = mine[k], ref[k].reshape(mine[k].shape)
            assert util.rel_inf(a, b) <= GRAD_TOL, f"{k}: rel_inf {util.rel_inf(a, b)}"


def test_wide_strip_fused_mask_equals_api_mask():
    """65552 x 32 px = 4097 x 2 tiles, ~20k small splats, some beyond x = 65536 (tile x >= 4096): the fused path's warp-cooperative
    tile mask, the API path's per-lane mask and (where built) the reference's kernels give the same lists and the same image"""
    W, H, n = 65552, 32, 20000
    rng = np.random.default_rng(3)
    px = np.concatenate([rng.uniform(0, W - 1, n - 2000), rng.uniform(65536, W - 1, 2000)])
    py = rng.uniform(0, H - 1, n)
    theta = rng.uniform(0, np.pi, n)
    raw = _leaves(W, H, px, py, theta, rng.uniform(0.5, 6.0, n), rng.uniform(0.3, 2.0, n), rng)
    raw["opacity"] = rng.uniform(-3.0, 3.0, (n, 1)).astype(np.float32)
    act = _activated(raw)
    view = view_from_camera(camera_from_pose(np.eye(3), np.zeros(3), W, H, FOV), (0.0, 0.0, 0.0), DEG, 1.0)
    api = run_ours(view, act)
    fused = run_fused(view, raw)
    full = run_ours(view, act, tile_cull=False)
    tile, _ = _instances(full)
    assert (tile % ((W + 15) // 16) >= 4096).sum() > 500, "too few instances beyond tile column 4096"
    assert api["num_listed"] < full["num_listed"]
    _assert_same_lists(api, fused, "API vs fused")
    for k in ("color", "radii", "n_contrib", "final_T"):
        np.testing.assert_array_equal(fused[k], api[k], err_msg=k)
    for k in ("color", "radii", "final_T"):
        np.testing.assert_array_equal(full[k], api[k], err_msg=k)
    np.testing.assert_array_equal(_last_contributor(view, full), _last_contributor(view, api))
    if util.have_ref():
        ref = run_ref(view, act)
        for k in ("color", "radii", "n_contrib", "final_T"):
            np.testing.assert_array_equal(full[k], ref[k], err_msg=f"reference: {k}")
        for k in ("color", "radii", "final_T"):
            np.testing.assert_array_equal(fused[k], ref[k], err_msg=f"reference: {k}")
