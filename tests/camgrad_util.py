"""Float64 arbiter of the camera gradients (render(camera_grad=True), lgr_backward_raw_camera).  TEST INFRASTRUCTURE ONLY.

The C oracle (oracle/lgo.c) differentiates the Gaussians only, so the camera terms are restated here in float64 numpy from the same
per-Gaussian inputs the oracle's preprocess backward reads: dL/dmean2D and dL/dconic from its blend backward, and the view-direction
term of dL/dmean3D, taken from a second call of its preprocess backward with dL/dmean2D = dL/dconic = 0 (then dL/dmean3D is that term
alone, exactly).  Each camera term differentiates one line of the reference's forward:
  t = p V (camera-space mean, forward.cu:81 via computeCov2D) and the 1.3 tan(fov) clamp with its masks (backward.cu:183-201),
  T = J W with J at the clamped t (forward.cu:88-99): dL/dW = J^T dL/dT,
  h = p Pm and ndc = h_xy / (h_w + 1e-7) (forward.cu:200-202, backward.cu:370-387),
  dir = (p - c) / |p - c| of the SH colour (forward.cu:22-28).
tests/test_camera_grad_cpu.py checks the result against central finite differences of the float64 oracle forward."""
from __future__ import annotations

import numpy as np

from oracle.lgo import Oracle, View
from tests import util

# the 27 live entries: viewmatrix [4r + k] (k < 3), projmatrix [4r + k] (k in 0, 1, 3), campos [c]
VIEW_LIVE = [4 * r + k for r in range(4) for k in range(3)]
PROJ_LIVE = [4 * r + k for r in range(4) for k in (0, 1, 3)]


def camera_grads_core(view: View, means3D, cov3D, radii, dL_dmean2D, dL_dconic, sh_dir, dL_dz=None, exact_clamp=False) -> dict:
    """Camera gradients from per-Gaussian inputs (float64).  sh_dir: the view-direction term of dL/dmean3D [P,3]; dL_dz: optional
    [P] gradient with respect to each Gaussian's view-space depth t_2 (the depth plane).  Only Gaussians with radii > 0 contribute.
    exact_clamp=False is the definition (the reference's, which the kernels follow); True is the exact derivative of the forward for
    Gaussians beyond the 1.3 tan(fov) clamp, for finite-difference checks of views that have such Gaussians.
    Returns view [16], proj [16], campos [3] and the sums of the absolute per-Gaussian terms (abs_view, abs_proj, abs_campos)."""
    f = lambda a: np.asarray(a, np.float64)  # noqa: E731
    vis = np.asarray(radii) > 0
    p3 = f(means3D)[vis]
    n = p3.shape[0]
    V, Pm = f(view.viewmatrix).reshape(4, 4), f(view.projmatrix).reshape(4, 4)
    c3 = f(cov3D).reshape(-1, 6)[vis]
    g2 = f(dL_dmean2D).reshape(-1, 2)[vis]
    dcon = f(dL_dconic).reshape(-1, 3)[vis]
    p = np.concatenate([p3, np.ones((n, 1))], 1)                              # [n,4]
    fx, fy = view.W / (2.0 * view.tanfovx), view.H / (2.0 * view.tanfovy)
    t = p @ V[:, :3]                                                          # t_k = sum_r p_r V[r][k]
    tz = t[:, 2]
    limx, limy = 1.3 * view.tanfovx, 1.3 * view.tanfovy
    txtz, tytz = t[:, 0] / tz, t[:, 1] / tz
    txc, tyc = np.clip(txtz, -limx, limx) * tz, np.clip(tytz, -limy, limy) * tz
    J = np.zeros((n, 2, 3))
    J[:, 0, 0], J[:, 0, 2] = fx / tz, -fx * txc / tz ** 2
    J[:, 1, 1], J[:, 1, 2] = fy / tz, -fy * tyc / tz ** 2
    T = J @ V[:3, :3].T[None]                                                 # T[i][r] = sum_k J[i][k] V[r][k]
    S = np.zeros((n, 3, 3))
    for (a, b), k in zip(((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)), range(6)):
        S[:, a, b] = S[:, b, a] = c3[:, k]
    C2 = T @ S @ T.transpose(0, 2, 1)
    a, b, c = C2[:, 0, 0] + 0.3, C2[:, 0, 1], C2[:, 1, 1] + 0.3
    dA, dB, dC = dcon[:, 0], dcon[:, 1], dcon[:, 2]
    denom = a * c - b * b
    d2 = 1.0 / (denom * denom + 1e-7)
    da = d2 * (-c * c * dA + 2 * b * c * dB + (denom - a * c) * dC)
    dc = d2 * (-a * a * dC + 2 * a * b * dB + (denom - a * c) * dA)
    db = d2 * 2 * (b * c * dA - (denom + 2 * b * b) * dB + a * b * dC)
    ST = S @ T.transpose(0, 2, 1)                                             # columns: S T0, S T1
    dT = np.zeros((n, 2, 3))
    dT[:, 0] = 2 * da[:, None] * ST[:, :, 0] + db[:, None] * ST[:, :, 1]
    dT[:, 1] = 2 * dc[:, None] * ST[:, :, 1] + db[:, None] * ST[:, :, 0]
    dJ = dT @ V[:3, :3]                                                       # dJ[i][k] = sum_r dT[i][r] V[r][k]
    xmul = ((txtz >= -limx) & (txtz <= limx)).astype(np.float64)
    ymul = ((tytz >= -limy) & (tytz <= limy)).astype(np.float64)
    dt = np.zeros((n, 3))
    dt[:, 0] = xmul * -fx / tz ** 2 * dJ[:, 0, 2]
    dt[:, 1] = ymul * -fy / tz ** 2 * dJ[:, 1, 2]
    # the reference treats the clamped t_x, t_y as constants in t_z (backward.cu:196-201); exact_clamp differentiates t_x = +-lim t_z
    kx, ky = (1 + xmul, 1 + ymul) if exact_clamp else (2.0, 2.0)
    dt[:, 2] = (-fx / tz ** 2 * dJ[:, 0, 0] - fy / tz ** 2 * dJ[:, 1, 1] + kx * fx * txc / tz ** 3 * dJ[:, 0, 2]
                + ky * fy * tyc / tz ** 3 * dJ[:, 1, 2])
    if dL_dz is not None:
        dt[:, 2] += f(dL_dz).reshape(-1)[vis]
    dW = J.transpose(0, 2, 1) @ dT                                            # dW[k][r] = sum_i J[i][k] dT[i][r] = dL/dV[r][k]
    termV = p[:, :, None] * dt[:, None, :]                                    # [n, r, k]
    termW = np.zeros((n, 4, 3))
    termW[:, :3, :] = dW.transpose(0, 2, 1)
    h = p @ Pm
    mw = 1.0 / (h[:, 3] + 1e-7)
    dh = np.stack([g2[:, 0] * mw, g2[:, 1] * mw, -(g2[:, 0] * h[:, 0] + g2[:, 1] * h[:, 1]) * mw * mw], 1)
    termP = p[:, :, None] * dh[:, None, :]
    termC = -f(sh_dir).reshape(-1, 3)[vis]
    out = dict(view=np.zeros(16), proj=np.zeros(16), campos=termC.sum(0), abs_view=np.zeros(16), abs_proj=np.zeros(16),
               abs_campos=np.abs(termC).sum(0))
    out["view"][VIEW_LIVE] = (termV + termW).sum(0).ravel()
    out["abs_view"][VIEW_LIVE] = (np.abs(termV) + np.abs(termW)).sum(0).ravel()
    out["proj"][PROJ_LIVE] = termP.sum(0).ravel()
    out["abs_proj"][PROJ_LIVE] = np.abs(termP).sum(0).ravel()
    return out


def sh_direction_term(o: Oracle, view: View, means3D, radii, clamped3, cov3D, dL_dcolor, shs, scales, rotations):
    """the view-direction term of the oracle's dL/dmean3D: its preprocess backward with dL/dmean2D = dL/dconic = 0"""
    P = np.asarray(means3D).shape[0]
    g3 = o.preprocess_backward(view, means3D, radii, clamped3, cov3D, np.zeros((P, 2)), np.zeros((P, 3)), dL_dcolor, shs=shs,
                               scales=scales, rotations=rotations)
    return g3["dL_dmeans3D"]


def camera_grads_oracle_forward(o: Oracle, view: View, fwd: dict, dpix, means3D, shs, scales, rotations, dL_dz=None,
                                exact_clamp=False) -> dict:
    """camera gradients of sum(dpix * image) (+ sum_i dL_dz_i t2_i) on the float64 oracle's own forward `fwd` (Oracle.forward)"""
    geom = fwd["geom"]
    P = geom["radii"].shape[0]
    g2 = o.blend_backward(view, P, fwd["ranges"], fwd["point_list"], geom["means2D"], geom["conic_opacity"], fwd["colors"],
                          fwd["final_T"], fwd["n_contrib"], dpix)
    sh = sh_direction_term(o, view, means3D, geom["radii"], geom["clamped"], geom["cov3D"], g2["dL_dcolor"], shs, scales, rotations)
    return camera_grads_core(view, means3D, geom["cov3D"], geom["radii"], g2["dL_dmean2D"], g2["dL_dconic"], sh, dL_dz, exact_clamp)


def camera_grads_float64(view: View, raw: dict, state: dict, dpix, act=None, extra2d=None, dL_dz=None) -> dict:
    """Exact camera gradients for the upstream gradient `dpix` on a given forward state (read_state() of the fused forward), next to
    util.leaf_grads_float64.  extra2d: optional (dL_dmean2D, dL_dconic) of a further blend backward to add (the depth / alpha
    planes' call); dL_dz: optional [P] gradient of each Gaussian's view-space depth."""
    act = util.activate(raw, view.sh_degree) if act is None else act
    o = Oracle(double=True)
    geom = state["geom"]
    P = act["means3D"].shape[0]
    clamped3 = np.stack([(geom["clamped_bits"] >> c) & 1 for c in range(3)], axis=1).astype(np.uint8)
    g2 = o.blend_backward(view, P, state["ranges"], state["point_list"], geom["means2D"], geom["conic_opacity"], geom["rgb"],
                          state["final_T"], state["n_contrib"], np.asarray(dpix, np.float32))
    sh = sh_direction_term(o, view, act["means3D"], state["radii"], clamped3, geom["cov3D"], g2["dL_dcolor"], act["shs"], act["scales"],
                           act["rotations"])
    m2, con = np.asarray(g2["dL_dmean2D"], np.float64), np.asarray(g2["dL_dconic"], np.float64)
    if extra2d is not None:
        m2, con = m2 + np.asarray(extra2d[0], np.float64), con + np.asarray(extra2d[1], np.float64)
    return camera_grads_core(view, act["means3D"], geom["cov3D"], state["radii"], m2, con, sh, dL_dz)
