"""Camera gradients, CPU: the float64 arbiter (tests/camgrad_util.py) against central finite differences of the float64 oracle forward,
entry by entry for the 27 live entries of viewmatrix, projmatrix and campos, on the scene of
test_oracle.py::test_backward_matches_finite_differences_in_double and the seeded configs of tests/util.py, with that test's acceptance
(median relative error < 1e-6, max < 1e-3); one case with a depth-plane term; the eight unread entries exactly 0; and a 6-DoF pose
chain (V, V @ K, inv(V)[3, :3]) applied to the arbiter's gradients against finite differences in the pose."""
import numpy as np
import pytest
import torch

from oracle.lgo import Oracle, View
from lightgaussian_b200.synth import make_cameras, make_scene
from tests.camgrad_util import PROJ_LIVE, VIEW_LIVE, camera_grads_oracle_forward
from tests.util import CONFIGS, make_config


def _fd_scene():
    P, W, H = 60, 48, 40
    sc = make_scene(P, scale_mult=0.5)
    a = {k: v.astype(np.float64) for k, v in sc["act"].items()}
    cam = make_cameras(5, W, H)[2]
    v = View(W, H, cam.tanfovx, cam.tanfovy, cam.world_view_transform.astype(np.float64), cam.full_proj_transform.astype(np.float64),
             cam.camera_center.astype(np.float64), np.array([0.2, 0.5, 0.7]), 3, 1.3)
    dpix = np.random.default_rng(1).standard_normal((3, H, W))
    return a, v, dpix


def _config_scene(name):
    """the config's scene and view in float64, opacities capped at 0.98: the reference's blend clamps alpha at 0.99 and its backward
    (like the oracle's, for the leaves as for the camera) does not differentiate that clamp, so a pair at the clamp makes the analytical
    gradient differ from the forward's finite differences at the 1e-4 level (the configs have opacities up to 0.999)"""
    act, v32, dpix = make_config(name)
    a = {k: np.asarray(x, np.float64) for k, x in act.items()}
    a["opacities"] = np.minimum(a["opacities"], 0.98)
    v = View(v32.W, v32.H, v32.tanfovx, v32.tanfovy, v32.viewmatrix.astype(np.float64), v32.projmatrix.astype(np.float64),
             v32.campos.astype(np.float64), v32.bg.astype(np.float64), v32.sh_degree, v32.scale_modifier)
    return a, v, dpix.astype(np.float64)


def _with(v, **kw):
    return View(v.W, v.H, v.tanfovx, v.tanfovy, kw.get("viewmatrix", v.viewmatrix), kw.get("projmatrix", v.projmatrix),
                kw.get("campos", v.campos), v.bg, v.sh_degree, v.scale_modifier)


class _Problem:
    """L(V, Pm, c) = sum(dpix * image) + sum_i wz_i t2_i (the depth term over the Gaussians visible in the base view, when wz is set)"""

    def __init__(self, a, v, dpix, depth_weights=False):
        self.o, self.a, self.v, self.dpix = Oracle(double=True), a, v, dpix
        self.fwd = self.forward(v)
        radii = self.fwd["geom"]["radii"]
        self.vis = radii > 0
        self.wz = None
        if depth_weights:
            self.wz = np.where(self.vis, np.random.default_rng(5).standard_normal(radii.shape[0]), 0.0)

    def forward(self, v):
        a = self.a
        return self.o.forward(v, a["means3D"], a["opacities"], shs=a["shs"], scales=a["scales"], rotations=a["rotations"])

    def loss(self, v):
        L = float((self.forward(v)["color"] * self.dpix).sum())
        if self.wz is not None:
            p = np.concatenate([self.a["means3D"], np.ones((self.a["means3D"].shape[0], 1))], 1)
            L += float((self.wz * (p @ np.asarray(v.viewmatrix).reshape(4, 4)[:, 2])).sum())
        return L

    def grads(self, exact_clamp=False):
        a = self.a
        return camera_grads_oracle_forward(self.o, self.v, self.fwd, self.dpix, a["means3D"], a["shs"], a["scales"], a["rotations"],
                                           dL_dz=self.wz, exact_clamp=exact_clamp)

    def fd(self, which, j):
        key = {"view": "viewmatrix", "proj": "projmatrix", "campos": "campos"}[which]

        def at(delta):
            arr = np.array(getattr(self.v, key), np.float64)
            arr.reshape(-1)[j] += delta
            return self.loss(_with(self.v, **{key: arr}))
        return smooth_fd(at)


def smooth_fd(at):
    """central difference of at(delta) at 0 with the first step (1e-6 down to 1e-8) that straddles no discrete decision of the forward:
    with 1000+ Gaussians a radius, tile or depth-order flip can lie within 1e-6 of the base view, and then the difference quotient at
    step h and at h/2 disagree (the jump divided by the step).  Discrete decisions are constant in the analytical gradient."""
    for h in (1e-6, 3e-7, 1e-7, 3e-8, 1e-8):
        a, b = (at(h) - at(-h)) / (2 * h), (at(h / 2) - at(-h / 2)) / h
        if abs(a - b) <= 1e-5 * (abs(a) + abs(b)) + 1e-9:
            return a
    return a


def _check_fd(prob, exact_clamp=False):
    g = prob.grads(exact_clamp)
    errs = []
    for which, live in (("view", VIEW_LIVE), ("proj", PROJ_LIVE), ("campos", range(3))):
        for j in live:
            num, ana = prob.fd(which, j), g[which][j]
            errs.append(abs(num - ana) / (abs(num) + abs(ana) + 1e-9))
    assert len(errs) == 27
    assert np.median(errs) < 1e-6, errs
    assert max(errs) < 1e-3, errs
    return g


def test_camera_grads_match_finite_differences_on_the_oracle_scene():
    prob = _Problem(*_fd_scene())
    assert prob.vis.sum() > 40
    _check_fd(prob)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_camera_grads_match_finite_differences_on_the_seeded_configs(name):
    """the "inside" camera sees Gaussians beyond the 1.3 tan(fov) clamp, whose t_z term the definition (the reference's backward) takes
    with the clamped t_x held constant; there the finite differences are compared with the clamp differentiated exactly, and the
    definition must differ from that only in the t_z column of V"""
    prob = _Problem(*_config_scene(name))
    clamped = name == "inside"
    g = _check_fd(prob, exact_clamp=clamped)
    if clamped:
        d = prob.grads()
        assert not np.allclose(d["view"], g["view"])
        np.testing.assert_array_equal(np.delete(d["view"], [2, 6, 10, 14]), np.delete(g["view"], [2, 6, 10, 14]))
        np.testing.assert_array_equal(d["proj"], g["proj"])
        np.testing.assert_array_equal(d["campos"], g["campos"])


def test_camera_grads_with_a_depth_term_match_finite_differences():
    _check_fd(_Problem(*_fd_scene(), depth_weights=True))


def test_unread_entries_are_exactly_zero():
    prob = _Problem(*_fd_scene(), depth_weights=True)
    g = prob.grads()
    for which, live, n in (("view", VIEW_LIVE, 16), ("proj", PROJ_LIVE, 16)):
        dead = [j for j in range(n) if j not in live]
        assert len(dead) == 4
        for j in dead:
            assert g[which][j] == 0.0 and g["abs_" + which][j] == 0.0
            assert prob.fd(which, j) == 0.0     # neither the forward nor the depth term reads V[4r+3] or Pm[4r+2]


def _hat(w):
    z = torch.zeros((), dtype=w.dtype)
    return torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])


def make_w2c_T(pose, R0, t0):
    """[4,4] transposed world-to-camera of the base pose (R0, t0) composed with the se(3) delta pose = (omega, tau):
    R = exp(omega^) R0, t = exp(omega^) t0 + tau; returned as the transposed matrix world_view_transform uses."""
    Rd = torch.linalg.matrix_exp(_hat(pose[:3]))
    R, t = Rd @ R0, Rd @ t0 + pose[3:]
    top = torch.cat([R, t[:, None]], 1)
    W2C = torch.cat([top, torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=pose.dtype)], 0)
    return W2C.T


def test_pose_chain_matches_finite_differences():
    """pose -> (V, V @ K, inv(V)[3, :3]) in float64 torch; the arbiter's three gradients pulled back through it equal finite differences
    of the oracle loss in the 6 pose parameters"""
    a, v, dpix = _fd_scene()
    V0 = torch.from_numpy(np.asarray(v.viewmatrix, np.float64))
    K = torch.linalg.inv(V0) @ torch.from_numpy(np.asarray(v.projmatrix, np.float64))
    R0, t0 = V0.T[:3, :3].clone(), V0.T[:3, 3].clone()

    def cams(pose):
        V = make_w2c_T(pose, R0, t0)
        return V, V @ K, torch.linalg.inv(V)[3, :3]

    def view_of(pose):
        with torch.no_grad():
            V, Pm, c = cams(pose)
        return _with(v, viewmatrix=V.numpy().copy(), projmatrix=Pm.numpy().copy(), campos=c.numpy().copy())

    pose0 = torch.zeros(6, dtype=torch.float64)
    prob = _Problem(a, view_of(pose0), dpix)
    g = prob.grads()
    pose = pose0.clone().requires_grad_(True)
    V, Pm, c = cams(pose)
    torch.autograd.backward([V, Pm, c], [torch.from_numpy(g["view"].reshape(4, 4)), torch.from_numpy(g["proj"].reshape(4, 4)),
                                         torch.from_numpy(g["campos"])])
    ana = pose.grad.numpy()
    errs = []
    for j in range(6):
        def at(h):
            d = torch.zeros(6, dtype=torch.float64)
            d[j] = h
            return prob.loss(view_of(pose0 + d))
        num = smooth_fd(at)
        errs.append(abs(num - ana[j]) / (abs(num) + abs(ana[j]) + 1e-9))
    assert np.median(errs) < 1e-6, errs
    assert max(errs) < 1e-3, errs
