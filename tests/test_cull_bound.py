"""The exact-culling predicate (lgr::rect_culled in lightgaussian_b200/csrc/lgr_math.cuh, used by the binning-time tile mask and the
round-1 blend kernels' sub-tile cull) compiled for the host and swept over far needle splats, where q = hA dx^2 + hC dy^2 + B dx dy
cancels terms of 1e5-1e7 down to values near the alpha threshold:
  - it never culls a rectangle in which the reference's pinned pair_power blends a pixel (o * exp(power) >= 1/255),
  - the rounding error of its q, relative to the mag it scales the margin by, stays under that margin's constant (LGR_CULL_REL),
with its operations pinned as the kernels compile them and with a host compiler free to contract them into FMAs."""
import ctypes as C
import os
import platform
import re
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "math_host.cpp")
HDR = os.path.join(os.path.dirname(HERE), "lightgaussian_b200", "csrc", "lgr_math.cuh")
FLAGS = ["-O2", "-fno-fast-math", "-shared", "-fPIC", "-std=c++17"]


def _cull_rel():
    return float(re.search(r"#define LGR_CULL_REL ([0-9.e+-]+)f", open(HDR).read()).group(1))


def _cpu_has_fma():
    if platform.machine() in ("aarch64", "arm64"):
        return True
    try:
        return re.search(r"^flags\s*:.*\bfma\b", open("/proc/cpuinfo").read(), re.M) is not None
    except OSError:
        return False


def _build(name, extra):
    lib = os.path.join(HERE, "native", "_build", name)
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        os.makedirs(os.path.dirname(lib), exist_ok=True)
        subprocess.check_call(["g++", *FLAGS, *extra, SRC, "-o", lib])
    return C.CDLL(lib)


@pytest.fixture(scope="module")
def pinned():
    """the pinned build (no contraction): the reference's pair_power exactly as the kernels evaluate it"""
    return _build("libmath_host.so", ["-ffp-contract=off"])


@pytest.fixture(scope="module", params=["no_contraction", "fma_contraction"])
def cull(request, pinned):
    if request.param == "no_contraction":
        return pinned
    if not _cpu_has_fma():
        pytest.skip("host CPU has no FMA instructions")
    extra = ["-ffp-contract=fast"] + (["-mfma"] if platform.machine() in ("x86_64", "AMD64") else [])
    return _build("libmath_host_fma.so", extra)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _needles(n, seed):
    """n far needles, each with one pixel rectangle (a 16 x 16 tile, or a border-clipped part of one) that its long axis passes near:
    screen sigma_major 200-2000 px, sigma_minor <= 0.3 px (plus the 0.3 px^2 low-pass), centres 100-1500 px from the rectangle, angles
    over the whole half-turn; a quarter at 45 degrees with integer centres (the edge minimiser then lies on a pixel centre).
    Returns float32 px, py, A, B, C (the conic) and int32 inclusive pixel bounds x0, x1, y0, y1."""
    rng = np.random.default_rng(seed)
    tx, ty = rng.integers(0, 128, n), rng.integers(0, 8, n)
    x0, y0 = 16 * tx, 16 * ty
    w = np.where(rng.random(n) < 0.25, rng.integers(1, 16, n), 16)      # clipped by an image border
    h = np.where(rng.random(n) < 0.25, rng.integers(1, 16, n), 16)
    x1, y1 = x0 + w - 1, y0 + h - 1
    theta = rng.uniform(0.0, np.pi, n)
    diag = rng.random(n) < 0.25
    theta[diag] = np.pi / 4 + np.pi / 2 * rng.integers(0, 2, diag.sum())
    d = rng.uniform(100.0, 1500.0, n)
    side = np.where(rng.random(n) < 0.5, 1.0, -1.0)
    # a target point in (or just outside) the rectangle on the needle's axis, the centre d px away along the axis
    txp = x0 + rng.uniform(-2.0, w + 1.0)
    typ = y0 + rng.uniform(-2.0, h + 1.0)
    perp = rng.uniform(-1.5, 1.5, n)
    cx = txp + side * d * np.cos(theta) - perp * np.sin(theta)
    cy = typ + side * d * np.sin(theta) + perp * np.cos(theta)
    cx[diag], cy[diag] = np.round(cx[diag]), np.round(cy[diag])
    sM = d / rng.uniform(0.4, 3.5, n)
    sM = np.clip(sM, 200.0, 2000.0)
    sm = rng.uniform(0.0, 0.3, n)
    c, s = np.cos(theta), np.sin(theta)
    a = c * c * sM * sM + s * s * sm * sm + 0.3
    b = c * s * (sM * sM - sm * sm)
    cc = s * s * sM * sM + c * c * sm * sm + 0.3
    det = a * cc - b * b
    f32 = lambda v: np.ascontiguousarray(v, np.float32)  # noqa: E731
    i32 = lambda v: np.ascontiguousarray(v, np.int32)  # noqa: E731
    return dict(px=f32(cx), py=f32(cy), A=f32(cc / det), B=f32(-b / det), C=f32(a / det), x0=i32(x0), x1=i32(x1), y0=i32(y0), y1=i32(y1))


def _max_power(lib, g):
    n = g["px"].size
    out = np.empty(n, np.float32)
    lib.mh_rect_max_power(n, *[_p(g[k]) for k in ("px", "py", "A", "B", "C", "x0", "x1", "y0", "y1")], _p(out))
    return out


def _cull(lib, g, o):
    n = g["px"].size
    culled, q, mag = np.empty(n, np.uint8), np.empty(n, np.float32), np.empty(n, np.float32)
    o = np.ascontiguousarray(o, np.float32)
    lib.mh_rect_cull(n, *[_p(g[k]) for k in ("px", "py", "A", "B", "C")], _p(o), *[_p(g[k]) for k in ("x0", "x1", "y0", "y1")],
                     _p(culled), _p(q), _p(mag))
    return culled.astype(bool), q, mag


def _qmin64(g):
    """the smallest q over the continuous rectangle, in float64 from the same float32 conic and centre"""
    f = lambda k: g[k].astype(np.float64)  # noqa: E731
    A, B, Cc, px, py = f("A"), f("B"), f("C"), f("px"), f("py")
    dx_lo, dx_hi, dy_lo, dy_hi = px - f("x1"), px - f("x0"), py - f("y1"), py - f("y0")
    cx, cy = np.clip(0.0, dx_lo, dx_hi), np.clip(0.0, dy_lo, dy_hi)
    q = lambda dx, dy: 0.5 * (A * dx * dx + Cc * dy * dy) + B * dx * dy  # noqa: E731
    qx = np.where(cx != 0, q(cx, np.clip(-B * cx / Cc, dy_lo, dy_hi)), np.inf)
    qy = np.where(cy != 0, q(np.clip(-B * cy / A, dx_lo, dx_hi), cy), np.inf)
    return np.minimum(qx, qy)


N_NEEDLES = 1 << 20


def test_far_needles_never_cull_a_blending_rectangle(pinned, cull):
    g = _needles(N_NEEDLES, seed=20261016)
    pmax = _max_power(pinned, g).astype(np.float64)
    G = np.exp(pmax)
    at = (G > 1e-3) & (G < 0.9)
    rng = np.random.default_rng(7)
    eps = rng.choice([1e-3, 5e-3, 2e-2], N_NEEDLES)
    # opacity that puts the reference's best pixel in the rectangle at alpha (1 + eps) / 255: it blends, the rectangle must be kept
    o_on = np.where(at, (1.0 + eps) / (255.0 * np.where(at, G, 1.0)), 0.5).astype(np.float32)
    sel = at & (o_on < 1.0)
    assert sel.sum() > 500_000, f"only {sel.sum()} needles have a rectangle at the threshold"
    gs = {k: v[sel] for k, v in g.items()}
    o_on = o_on[sel]
    blends = o_on.astype(np.float64) * np.exp(pmax[sel]) >= (1.0 / 255.0) * (1.0 - 1e-6)
    assert blends.all()
    culled, q, mag = _cull(cull, gs, o_on)
    bad = np.flatnonzero(culled & blends)
    assert bad.size == 0, (f"{bad.size} of {blends.sum()} rectangles culled although the reference blends a pixel in them; worst q - thr: "
                           f"{float(np.max(q[bad] - np.log(257.55 * o_on[bad].astype(np.float64)))):.3g}, mag up to {float(mag[bad].max()):.3g}")
    # the margin's constant covers the rounding of q, with room for the reference's own rounding of power at the pixel
    err = np.abs(q.astype(np.float64) - _qmin64(gs)) / np.maximum(mag.astype(np.float64), 1e-30)
    rel = _cull_rel()
    assert float(err.max()) < 0.5 * rel, f"q rounding {float(err.max()):.3g} x mag (constant {rel:g})"
    assert float(np.median(mag)) > 1e4, "the sweep does not reach the cancelling regime"
    # not vacuous: with the best pixel at about half the threshold alpha, a good share of the same rectangles is culled
    o_off = (o_on.astype(np.float64) * 0.5 / (1.0 + 2e-2)).astype(np.float32)
    culled_off, _, _ = _cull(cull, gs, o_off)
    assert culled_off.mean() > 0.25, f"only {culled_off.mean():.3f} of the below-threshold rectangles are culled"


def test_bare_alpha_margin_fails_on_the_sweep(pinned):
    """The 1 % alpha margin alone (q > thr, no mag term) culls rectangles the reference blends in on the same sweep: the sweep reaches
    the cancellation the LGR_CULL_REL term exists for."""
    g = _needles(1 << 18, seed=20261017)
    pmax = _max_power(pinned, g).astype(np.float64)
    G = np.exp(pmax)
    sel = (G > 1e-3) & (G < 0.9) & ((1.0 + 1e-3) / (255.0 * np.where(G > 0, G, 1.0)) < 1.0)
    gs = {k: v[sel] for k, v in g.items()}
    o = ((1.0 + 1e-3) / (255.0 * G[sel])).astype(np.float32)
    _, q, mag = _cull(pinned, gs, o)
    thr = np.log(np.float32(257.55) * o).astype(np.float32)
    assert ((q > thr) & (q < thr + np.float32(_cull_rel()) * mag)).sum() > 0
