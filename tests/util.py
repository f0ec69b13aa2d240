"""Shared helpers for the parity tests: scene/view construction, running our CUDA path and (when present)
the reference's own kernels through oracle/_ref, and comparison metrics."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from lightgaussian_b200.synth import make_scene, make_cameras, inside_camera  # noqa: F401
from oracle.lgo import Oracle, View

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_rasterizer.so")


def view_from_camera(cam, bg=(0.0, 0.0, 0.0), sh_degree=3, scale_modifier=1.0) -> View:
    return View(cam.image_width, cam.image_height, cam.tanfovx, cam.tanfovy, cam.world_view_transform, cam.full_proj_transform,
                cam.camera_center, np.asarray(bg, np.float32), sh_degree, scale_modifier)


# name -> (P, W, H, camera factory, sh_degree, bg, scale_modifier, seed, scale_mult)
CONFIGS = {
    "outside": dict(P=1500, W=170, H=130, cam="sphere", deg=3, bg=(0.0, 0.0, 0.0), mod=1.0, seed=11, scale_mult=1.5),
    "inside": dict(P=1500, W=160, H=112, cam="inside", deg=2, bg=(1.0, 1.0, 1.0), mod=1.3, seed=12, scale_mult=1.0),
    "deg1": dict(P=1000, W=96, H=64, cam="sphere", deg=1, bg=(0.2, 0.5, 0.7), mod=1.0, seed=13, scale_mult=2.0),
    "deg0": dict(P=1000, W=64, H=96, cam="sphere", deg=0, bg=(0.0, 0.0, 0.0), mod=0.7, seed=14, scale_mult=3.0),
}


def make_config(name):
    c = CONFIGS[name]
    scene = make_scene(c["P"], sh_degree=3, seed=c["seed"], scale_mult=c["scale_mult"])
    cam = inside_camera(c["W"], c["H"]) if c["cam"] == "inside" else make_cameras(5, c["W"], c["H"])[2]
    view = view_from_camera(cam, c["bg"], c["deg"], c["mod"])
    rng = np.random.default_rng(c["seed"] + 1000)
    dL_dpix = rng.standard_normal((3, c["H"], c["W"])).astype(np.float32)
    return scene["act"], view, dL_dpix


# ------------------------------------------------------------------------------------------------
# our CUDA path, with every intermediate read back
# ------------------------------------------------------------------------------------------------
def _t(a, device="cuda"):
    import torch
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(device)


def _empty():
    import torch
    return torch.Tensor([])


def run_ours(view: View, act: dict, count=False, dL_dpix=None, colors_precomp=None, cov3D_precomp=None, debug=False, tile_cull=True,
             blend_mode=0, bin_mode=None):
    """tile_cull=False makes the per-tile lists identical to the reference's (needed to compare point_list / ranges /
    n_contrib); the product default (True) lists only instances that can contribute."""
    import torch
    from lightgaussian_b200 import capi
    from lightgaussian_b200.rasterizer import _C
    dev = "cuda"
    capi.set_tile_culling(tile_cull)
    capi.set_blend_mode(blend_mode)      # 0 = ring kernels (the product default), 1 = the round-1 kernels
    capi.set_binning_mode(capi.DEFAULT_BINNING_MODE if bin_mode is None else bin_mode)   # 2 = library sorts (default); 0 / 1 = hand-written
    try:
        return _run_ours(view, act, count, dL_dpix, colors_precomp, cov3D_precomp, debug)
    finally:
        capi.set_tile_culling(True)
        capi.set_blend_mode(0)
        capi.set_binning_mode(capi.DEFAULT_BINNING_MODE)


def _run_ours(view, act, count, dL_dpix, colors_precomp, cov3D_precomp, debug):
    import torch
    from lightgaussian_b200 import capi
    from lightgaussian_b200.rasterizer import _C
    dev = "cuda"
    means3D, opac = _t(act["means3D"]), _t(act["opacities"])
    shs = _empty() if colors_precomp is not None else _t(act["shs"])
    colors = _t(colors_precomp) if colors_precomp is not None else _empty()
    scales = _empty() if cov3D_precomp is not None else _t(act["scales"])
    rots = _empty() if cov3D_precomp is not None else _t(act["rotations"])
    cov = _t(cov3D_precomp) if cov3D_precomp is not None else _empty()
    bg, vm, pm, cp = _t(view.bg), _t(view.viewmatrix), _t(view.projmatrix), _t(view.campos)
    args = (bg, means3D, colors, opac, scales, rots, view.scale_modifier, cov, vm, pm, view.tanfovx, view.tanfovy, view.H, view.W, shs,
            view.sh_degree, cp, False, debug)
    out = {}
    if count:
        cnt, score, R, color, radii, geom, binning, img = _C.count_gaussians(*args, True)
        out["gaussians_count"], out["important_score"] = cnt.cpu().numpy(), score.cpu().numpy()
    else:
        R, color, radii, geom, binning, img = _C.rasterize_gaussians(*args)
    P = means3D.shape[0]
    out.update(num_rendered=R, color=color.cpu().numpy(), radii=radii.cpu().numpy())
    if P > 0:
        out.update(read_state(view, P, R, out["radii"], geom, binning, img))
    if dL_dpix is not None and not count:
        g = _C.rasterize_gaussians_backward(bg, means3D, radii, colors, scales, rots, view.scale_modifier, cov, vm, pm, view.tanfovx,
                                            view.tanfovy, _t(dL_dpix), shs, view.sh_degree, cp, geom, R, binning, img, debug)
        names = ["dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales", "dL_drotations"]
        out["grads"] = {n: t.cpu().numpy() for n, t in zip(names, g)}
    torch.cuda.synchronize()
    return out


def read_state(view: View, P, R, radii, geom, binning, img) -> dict:
    """The forward state a backward reads, copied out of the three blobs of a forward (plain or fused: same layouts)."""
    from lightgaussian_b200 import capi
    gl, _ = capi.geometry_layout(P)
    il, _ = capi.image_layout(view.W, view.H)
    gb, ib, bb = geom.cpu().numpy(), img.cpu().numpy(), binning.cpu().numpy()
    hdr = np.frombuffer(gb, dtype=np.int32, count=2, offset=0)
    assert int(hdr[1]) == R, (hdr, R)                 # header[1] = the reference's num_rendered
    n_listed = int(hdr[0])                            # header[0] = instances actually listed (<= R)
    bl, _ = capi.binning_layout(n_listed, view.W, view.H)
    N = view.W * view.H
    tiles = ((view.W + 15) // 16) * ((view.H + 15) // 16)

    def arr(buf, off, dtype, n):
        return np.frombuffer(buf, dtype=dtype, count=n, offset=off).copy()
    out = dict(num_listed=n_listed, radii=np.asarray(radii))
    out["geom"] = dict(
        depths=arr(gb, gl["depth"], np.float32, P), means2D=arr(gb, gl["means2D"], np.float32, 2 * P).reshape(P, 2),
        conic_opacity=arr(gb, gl["conic_opacity"], np.float32, 4 * P).reshape(P, 4),
        rgb=arr(gb, gl["rgb"], np.float32, 4 * P).reshape(P, 4)[:, :3].copy(),
        cov3D=arr(gb, gl["cov3D"], np.float32, 6 * P).reshape(P, 6), clamped_bits=arr(gb, gl["clamped"], np.uint8, P),
        tiles_touched=arr(gb, gl["tiles_touched"], np.uint32, P), sorted_ids=arr(gb, gl["sorted_ids"], np.uint32, P),
        radii=out["radii"])
    out["final_T"] = arr(ib, il["final_T"], np.float32, N)
    out["n_contrib"] = arr(ib, il["n_contrib"], np.uint32, N)
    out["ranges"] = arr(ib, il["ranges"], np.uint32, 2 * tiles).reshape(tiles, 2)
    out["point_list"] = arr(bb, bl["point_list"], np.uint32, n_listed) if n_listed > 0 else np.zeros(0, np.uint32)
    return out


# ------------------------------------------------------------------------------------------------
# the float64 oracle's backward on OUR forward state (so no threshold can differ)
# ------------------------------------------------------------------------------------------------
def oracle_backward_on_our_state(o, view, act, ours, dpix, colors=None, cov=None):
    geom = ours["geom"]
    P = act["means3D"].shape[0]
    clamped3 = np.stack([(geom["clamped_bits"] >> c) & 1 for c in range(3)], axis=1).astype(np.uint8)
    col = geom["rgb"] if colors is None else colors
    g2 = o.blend_backward(view, P, ours["ranges"], ours["point_list"], geom["means2D"], geom["conic_opacity"], col,
                          ours["final_T"], ours["n_contrib"], dpix)
    g3 = o.preprocess_backward(view, act["means3D"], ours["radii"], clamped3, geom["cov3D"] if cov is None else cov,
                               g2["dL_dmean2D"], g2["dL_dconic"], g2["dL_dcolor"],
                               shs=None if colors is not None else act["shs"],
                               scales=None if cov is not None else act["scales"],
                               rotations=None if cov is not None else act["rotations"])
    return g2, g3


LEAVES = ("xyz", "features_dc", "features_rest", "scaling", "rotation", "opacity")


def activate(raw: dict, sh_degree: int) -> dict:
    """The activated inputs the fused kernels compute from GaussianModel's raw leaves (exp / normalize / sigmoid, float32), with the
    SH rows cut to the (sh_degree+1)^2 coefficients the view uses."""
    M = (sh_degree + 1) ** 2
    rot = raw["rotation"].astype(np.float32)
    n = np.maximum(np.sqrt((rot * rot).sum(1, keepdims=True)), np.float32(1e-12))
    return dict(means3D=np.ascontiguousarray(raw["xyz"], np.float32), scales=np.exp(raw["scaling"]).astype(np.float32),
                rotations=(rot / n).astype(np.float32), opacities=(1.0 / (1.0 + np.exp(-raw["opacity"]))).astype(np.float32),
                shs=np.ascontiguousarray(np.concatenate([raw["features_dc"], raw["features_rest"]], axis=1)[:, :M], np.float32))


def leaf_grads_from_activated(raw: dict, g: dict) -> dict:
    """Chain rule of GaussianModel's activations, in float64: gradients with respect to the activated inputs (keys of
    Rasterizer::backward: dL_dmeans3D, dL_dsh, dL_dscales, dL_drotations, dL_dopacity, dL_dmeans2D) -> gradients of the six raw
    leaves and of viewspace_points ("means2D", [P, 3], z column zero)."""
    P, K = raw["xyz"].shape[0], raw["features_rest"].shape[1]
    f64 = lambda a: np.asarray(a, np.float64)  # noqa: E731
    dsh = f64(g["dL_dsh"]).reshape(P, -1, 3)
    rest = np.zeros((P, K, 3))
    rest[:, :dsh.shape[1] - 1] = dsh[:, 1:1 + K]
    v = f64(raw["rotation"])
    nv = np.maximum(np.sqrt((v * v).sum(1, keepdims=True)), 1e-12)
    q, gr = v / nv, f64(g["dL_drotations"]).reshape(P, 4)
    sig = 1.0 / (1.0 + np.exp(-f64(raw["opacity"])))
    m2 = np.zeros((P, 3))
    m2[:, :2] = f64(g["dL_dmeans2D"]).reshape(P, -1)[:, :2]
    return dict(xyz=f64(g["dL_dmeans3D"]).reshape(P, 3), features_dc=dsh[:, :1].copy(), features_rest=rest,
                scaling=f64(g["dL_dscales"]).reshape(P, 3) * np.exp(f64(raw["scaling"])),
                rotation=(gr - q * (q * gr).sum(1, keepdims=True)) / nv,
                opacity=f64(g["dL_dopacity"]).reshape(P, 1) * sig * (1.0 - sig), means2D=m2)


def leaf_grads_float64(view: View, raw: dict, state: dict, dpix, act=None) -> dict:
    """Exact (float64 oracle) gradients of the six raw leaves and of viewspace_points for the upstream gradient `dpix`, evaluated on a
    given forward state (read_state() of the fused forward), so that every threshold decision is the kernels' own.  `raw` holds the
    leaves as float32 numpy arrays, features_rest contiguous; view.sh_degree is the active degree.  `act`: the activated inputs the
    kernels saw (default: activate(raw))."""
    act = activate(raw, view.sh_degree) if act is None else act
    g2, g3 = oracle_backward_on_our_state(Oracle(double=True), view, act, state, np.asarray(dpix, np.float32))
    return leaf_grads_from_activated(raw, dict(dL_dmeans2D=g2["dL_dmean2D"], dL_dopacity=g2["dL_dopacity"], **g3))


def element_ratios(ours, exact, rho, alpha):
    """|ours - exact| / (rho |exact| + alpha max|exact|) per entry (float64); > 1 fails assert_every_element"""
    a, e = np.asarray(ours, np.float64).ravel(), np.asarray(exact, np.float64).ravel()
    assert a.shape == e.shape, (a.shape, e.shape)
    bound = rho * np.abs(e) + alpha * np.abs(e).max(initial=0.0)
    err = np.abs(a - e)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return np.where(np.isnan(a), np.inf, r)


def assert_every_element(ours, exact, rho, alpha, name):
    """|ours - exact| <= rho |exact| + alpha max|exact| for EVERY entry (no quantile).  Returns the worst ratio to the bound; on failure
    the message lists the worst entries."""
    r = element_ratios(ours, exact, rho, alpha)
    worst = float(r.max(initial=0.0))
    if worst > 1.0:
        a, e = np.asarray(ours, np.float64), np.asarray(exact, np.float64)
        bad = np.argsort(r)[::-1][:8]
        rows = [f"  {np.unravel_index(int(i), e.shape)}: ours {a.ravel()[i]:.9g}  exact {e.ravel()[i]:.9g}  ratio {r[i]:.3g}" for i in bad
                if r[i] > 1.0]
        raise AssertionError(f"{name}: {int((r > 1.0).sum())} of {r.size} entries outside {rho:g} |exact| + {alpha:g} max|exact| "
                             f"(max|exact| = {np.abs(e).max(initial=0.0):.3g}); worst:\n" + "\n".join(rows))
    return worst


# ------------------------------------------------------------------------------------------------
# the reference's own kernels (oracle/_ref/libref_rasterizer.so), GPU only
# ------------------------------------------------------------------------------------------------
def have_ref() -> bool:
    return os.path.exists(REF_LIB)


_ref_lib = None


def ref_lib():
    global _ref_lib
    if _ref_lib is None:
        lib = C.CDLL(REF_LIB)
        lib.ref_state_create.restype = C.c_void_p
        lib.ref_state_destroy.argtypes = [C.c_void_p]
        vp, i, f = C.c_void_p, C.c_int, C.c_float
        lib.ref_forward.restype = i
        lib.ref_forward.argtypes = [vp, i, i, i, i, vp, i, i, vp, vp, vp, vp, vp, f, vp, vp, vp, vp, vp, f, f, i, vp, vp, vp, vp]
        lib.ref_backward.restype = None
        lib.ref_backward.argtypes = [vp, i, i, i, vp, i, i, vp, vp, vp, vp, f, vp, vp, vp, vp, vp, f, f, vp, vp] + [vp] * 9
        lib.ref_geom_ptrs.argtypes = [vp, C.POINTER(vp)]
        lib.ref_image_ptrs.argtypes = [vp, i, C.POINTER(vp)]
        lib.ref_binning_ptrs.argtypes = [vp, C.POINTER(vp)]
        lib.ref_read.restype = i
        lib.ref_read.argtypes = [vp, vp, C.c_size_t]
        _ref_lib = lib
    return _ref_lib


def _dptr(t):
    return None if t is None else t.data_ptr()


def _from_dev(ptr, nbytes, dtype, shape):
    """copy `nbytes` from a raw device pointer into a numpy array"""
    host = np.empty(nbytes, np.uint8)
    err = ref_lib().ref_read(host.ctypes.data_as(C.c_void_p), ptr, nbytes)
    assert err == 0, f"cudaMemcpy failed: {err}"
    return host.view(dtype).reshape(shape).copy()


def run_ref(view: View, act: dict, count=False, dL_dpix=None, colors_precomp=None, cov3D_precomp=None):
    """Same outputs as run_ours(), produced by the reference's kernels."""
    import torch
    lib = ref_lib()
    st = lib.ref_state_create()
    try:
        means3D, opac = _t(act["means3D"]), _t(act["opacities"])
        shs = None if colors_precomp is not None else _t(act["shs"])
        colors = _t(colors_precomp)
        scales = None if cov3D_precomp is not None else _t(act["scales"])
        rots = None if cov3D_precomp is not None else _t(act["rotations"])
        cov = _t(cov3D_precomp)
        bg, vm, pm, cp = _t(view.bg), _t(view.viewmatrix), _t(view.projmatrix), _t(view.campos)
        P = means3D.shape[0]
        M = 0 if shs is None else shs.shape[1]
        W, H = view.W, view.H
        color = torch.zeros((3, H, W), dtype=torch.float32, device="cuda")
        radii = torch.zeros(P, dtype=torch.int32, device="cuda")
        cnt = torch.zeros(P, dtype=torch.int32, device="cuda")
        score = torch.zeros(P, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        R = lib.ref_forward(st, int(count), P, view.sh_degree, M, _dptr(bg), W, H, _dptr(means3D), _dptr(shs), _dptr(colors), _dptr(opac),
                            _dptr(scales), view.scale_modifier, _dptr(rots), _dptr(cov), _dptr(vm), _dptr(pm), _dptr(cp), view.tanfovx,
                            view.tanfovy, 0, _dptr(color), _dptr(radii), _dptr(cnt), _dptr(score))
        torch.cuda.synchronize()
        out = dict(num_rendered=R, color=color.cpu().numpy(), radii=radii.cpu().numpy())
        if count:
            out["gaussians_count"], out["important_score"] = cnt.cpu().numpy(), score.cpu().numpy()
        gp = (C.c_void_p * 7)()
        lib.ref_geom_ptrs(st, gp)
        ip = (C.c_void_p * 3)()
        lib.ref_image_ptrs(st, W * H, ip)
        bp = (C.c_void_p * 1)()
        lib.ref_binning_ptrs(st, bp)
        N = W * H
        tiles = ((W + 15) // 16) * ((H + 15) // 16)
        vis = out["radii"] > 0
        geom = dict(depths=_from_dev(gp[0], 4 * P, np.float32, (P,)), clamped=_from_dev(gp[1], 3 * P, np.uint8, (P, 3)),
                    means2D=_from_dev(gp[2], 8 * P, np.float32, (P, 2)), cov3D=_from_dev(gp[3], 24 * P, np.float32, (P, 6)),
                    conic_opacity=_from_dev(gp[4], 16 * P, np.float32, (P, 4)), rgb=_from_dev(gp[5], 12 * P, np.float32, (P, 3)),
                    tiles_touched=_from_dev(gp[6], 4 * P, np.uint32, (P,)), radii=out["radii"])
        for k in ("depths", "means2D", "conic_opacity", "rgb", "clamped"):  # rows of culled Gaussians are uninitialised in the reference
            geom[k][~vis] = 0
        out["geom"] = geom
        out["final_T"] = _from_dev(ip[0], 4 * N, np.float32, (N,))
        out["n_contrib"] = _from_dev(ip[1], 4 * N, np.uint32, (N,))
        out["ranges"] = _from_dev(ip[2], 8 * tiles, np.uint32, (tiles, 2))
        out["point_list"] = _from_dev(bp[0], 4 * R, np.uint32, (R,)) if R > 0 else np.zeros(0, np.uint32)
        if dL_dpix is not None and not count:
            z = lambda *s: torch.zeros(s, dtype=torch.float32, device="cuda")  # noqa: E731
            g = dict(dL_dmeans2D=z(P, 3), dL_dconic=z(P, 2, 2), dL_dopacity=z(P, 1), dL_dcolors=z(P, 3), dL_dmeans3D=z(P, 3),
                     dL_dcov3D=z(P, 6), dL_dsh=z(P, max(M, 0), 3), dL_dscales=z(P, 3), dL_drotations=z(P, 4))
            dp = _t(dL_dpix)
            torch.cuda.synchronize()
            lib.ref_backward(st, P, view.sh_degree, M, _dptr(bg), W, H, _dptr(means3D), _dptr(shs), _dptr(colors), _dptr(scales),
                             view.scale_modifier, _dptr(rots), _dptr(cov), _dptr(vm), _dptr(pm), _dptr(cp), view.tanfovx, view.tanfovy,
                             _dptr(radii), _dptr(dp), _dptr(g["dL_dmeans2D"]), _dptr(g["dL_dconic"]), _dptr(g["dL_dopacity"]),
                             _dptr(g["dL_dcolors"]), _dptr(g["dL_dmeans3D"]), _dptr(g["dL_dcov3D"]),
                             _dptr(g["dL_dsh"]) if M > 0 else None, _dptr(g["dL_dscales"]), _dptr(g["dL_drotations"]))
            torch.cuda.synchronize()
            out["grads"] = {k: v.cpu().numpy() for k, v in g.items()}
        return out
    finally:
        lib.ref_state_destroy(st)


# ------------------------------------------------------------------------------------------------
# metrics
# ------------------------------------------------------------------------------------------------
def rel_inf(a, b, eps=1e-12):
    """||a-b||_inf / max(||b||_inf, eps): the gradient parity metric of SURVEY.md section 8c."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max(initial=0.0) / max(np.abs(b).max(initial=0.0), eps))


def elem_rel(a, b, floor=1e-6):
    """Per-element relative error |a-b|/|b| on the entries with |b| > floor (SURVEY.md section 8c, second gradient metric).
    Returns (sorted errors, count); quantiles of it are what the tests bound -- the reference's own float atomics make single small
    entries differ run to run, so a max over millions of entries is not a stable statistic, its quantiles are."""
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    m = np.abs(b) > floor
    if not m.any():
        return np.zeros(0), 0
    e = np.sort(np.abs(a[m] - b[m]) / np.abs(b[m]))
    return e, int(m.sum())


def assert_elementwise(a, b, name, tol=1e-3, frac=0.995, median=2e-5, exact=None):
    """at least `frac` of the entries with |b| > 1e-6 agree to `tol` relative, and the median relative error is <= `median`.

    `exact` (optional) = the same gradient from the float64 oracle.  The reference's float atomics (backward.cu:523-541) make ITS
    small entries wander at the 1e-3 level from run to run on scenes with screen-filling splats, so there the arbiter is the exact
    value: our `frac` quantile of |a - exact| / |exact| must stay below `tol` or below 1.5x the reference's own quantile, and the
    direct comparison is bounded at 3 * tol."""
    e, n = elem_rel(a, b)
    if n == 0:
        return
    q = e[min(n - 1, int(frac * n))]
    if exact is not None:
        ea, na = elem_rel(a, exact)
        eb, nb = elem_rel(b, exact)
        qa, qb = ea[min(na - 1, int(frac * na))], eb[min(nb - 1, int(frac * nb))]
        assert qa <= max(tol, 1.5 * qb), (f"{name}: {100 * frac:.1f} % quantile of our per-element error against the float64 oracle is {qa:.2e} "
                                          f"(reference kernels: {qb:.2e}; n = {na})")
        assert q <= 3 * tol, f"{name}: {100 * frac:.1f} % quantile of the per-element relative error vs the reference is {q:.2e} (n = {n})"
    else:
        assert q <= tol, f"{name}: {100 * frac:.1f} % quantile of the per-element relative error is {q:.2e} (> {tol:g}; n = {n})"
    assert e[n // 2] <= median, f"{name}: median per-element relative error {e[n // 2]:.2e} (> {median:g})"


def rel_l2(a, b, eps=1e-30):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), eps))


def oracle_from_geometry(o: Oracle, view: View, geom: dict, count=False, want_fragile=True):
    """oracle binning + blend driven by a GIVEN per-Gaussian geometry (ours or the reference's)."""
    point_list, ranges = o.bin(view, geom["means2D"], geom["depths"], geom["radii"], geom["tiles_touched"])
    P = geom["radii"].shape[0]
    cnt = np.zeros(P, np.int64) if count else None
    img = o.blend_forward(view, ranges, point_list, geom["means2D"], geom["rgb"], geom["conic_opacity"], cnt, want_fragile)
    img.update(point_list=point_list, ranges=ranges, gaussians_count=cnt)
    return img
