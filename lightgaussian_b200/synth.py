"""Deterministic synthetic scenes and cameras (SURVEY.md section 8d) for tests and bench.py.

No dataset or checkpoint ships with the project, so every measurement uses a seeded random
Gaussian cloud and cameras on a Fibonacci sphere.  Camera matrices follow the reference's
convention exactly (scene/cameras.py:70-85, utils/graphics_utils.py:38-77): `world_view_transform`
and `full_proj_transform` are stored TRANSPOSED (row-vector convention), `camera_center` is row 3
of the inverse view transform.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List

import numpy as np


@dataclass
class SynthCamera:
    """The attributes gaussian_renderer.render() reads from a viewpoint camera
    (reference gaussian_renderer/__init__.py:49-62), as numpy arrays."""
    image_width: int
    image_height: int
    FoVx: float
    FoVy: float
    world_view_transform: np.ndarray  # [4,4] float32, transposed W2C
    full_proj_transform: np.ndarray   # [4,4] float32, transposed (Proj @ W2C)
    camera_center: np.ndarray         # [3] float32
    znear: float = 0.01
    zfar: float = 100.0

    @property
    def tanfovx(self) -> float:
        return math.tan(self.FoVx * 0.5)

    @property
    def tanfovy(self) -> float:
        return math.tan(self.FoVy * 0.5)


def projection_matrix(znear: float, zfar: float, fovx: float, fovy: float) -> np.ndarray:
    """Same frustum as utils/graphics_utils.py:51-77 (float32 arithmetic like torch.zeros(4,4))."""
    ty, tx = math.tan(fovy / 2), math.tan(fovx / 2)
    top, right = ty * znear, tx * znear
    bottom, left = -top, -right
    Pm = np.zeros((4, 4), np.float32)
    Pm[0, 0] = 2.0 * znear / (right - left)
    Pm[1, 1] = 2.0 * znear / (top - bottom)
    Pm[0, 2] = (right + left) / (right - left)
    Pm[1, 2] = (top + bottom) / (top - bottom)
    Pm[3, 2] = 1.0
    Pm[2, 2] = zfar / (zfar - znear)
    Pm[2, 3] = -(zfar * znear) / (zfar - znear)
    return Pm


def camera_from_pose(R_w2c: np.ndarray, t: np.ndarray, W: int, H: int, fovx: float, znear=0.01, zfar=100.0) -> SynthCamera:
    fovy = 2.0 * math.atan(math.tan(fovx / 2) * H / W)
    Rt = np.zeros((4, 4), np.float64)
    Rt[:3, :3] = R_w2c
    Rt[:3, 3] = t
    Rt[3, 3] = 1.0
    wvt = np.float32(Rt).T.copy()                       # transposed storage
    proj_t = projection_matrix(znear, zfar, fovx, fovy).T.copy()
    full = (wvt @ proj_t).astype(np.float32)            # == (Proj @ W2C)^T
    center = np.linalg.inv(wvt.astype(np.float64))[3, :3].astype(np.float32)
    return SynthCamera(W, H, fovx, fovy, np.ascontiguousarray(wvt), np.ascontiguousarray(full), np.ascontiguousarray(center),
                       znear, zfar)


def look_at(cam_pos, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    """W2C rotation / translation for a camera with x right, y down, z forward (COLMAP convention)."""
    c = np.asarray(cam_pos, np.float64)
    f = np.asarray(target, np.float64) - c
    f /= np.linalg.norm(f)
    u = np.asarray(up, np.float64)
    if abs(float(f @ u)) > 0.99:
        u = np.array([0.0, 1.0, 0.0])
    x = np.cross(f, u)
    x /= np.linalg.norm(x)
    y = np.cross(f, x)
    R = np.stack([x, y, f])
    return R, -R @ c


def make_cameras(n: int, W: int, H: int, fovx_deg: float = 60.0, radius: float = 3.0) -> List[SynthCamera]:
    """n poses on a Fibonacci sphere of the given radius, looking at the origin, up = +z."""
    cams = []
    golden = math.pi * (3.0 - math.sqrt(5.0))
    for i in range(n):
        z = 1.0 - 2.0 * (i + 0.5) / n
        r = math.sqrt(max(0.0, 1.0 - z * z))
        th = golden * i
        pos = radius * np.array([r * math.cos(th), r * math.sin(th), z])
        R, t = look_at(pos)
        cams.append(camera_from_pose(R, t, W, H, math.radians(fovx_deg)))
    return cams


def inside_camera(W: int, H: int, fovx_deg: float = 60.0) -> SynthCamera:
    """Correctness-only camera INSIDE the cloud, looking +x: exercises the z<=0.2 cull, the 1.3*tanfov
    clamp and very large splats (SURVEY.md section 8d, C1)."""
    R, t = look_at((0.3, 0.2, 0.1), target=(1.3, 0.2, 0.1))
    return camera_from_pose(R, t, W, H, math.radians(fovx_deg))


def make_scene(P: int, sh_degree: int = 3, seed: int = 0, scale_mult: float = 1.0) -> dict:
    """Raw (pre-activation) parameters with GaussianModel's layout (scene/gaussian_model.py:98-118) and the
    activated tensors render() feeds the rasterizer.  All float32, C-contiguous numpy."""
    rng = np.random.default_rng(seed)
    M = (sh_degree + 1) ** 2
    s0 = 0.6 * P ** (-1.0 / 3.0) * scale_mult
    raw = dict(
        xyz=rng.uniform(-1.0, 1.0, (P, 3)).astype(np.float32),
        scaling=(math.log(s0) + 0.5 * rng.standard_normal((P, 3))).astype(np.float32),
        rotation=rng.standard_normal((P, 4)).astype(np.float32),
        opacity=(2.0 * rng.standard_normal((P, 1))).astype(np.float32),
        features_dc=rng.standard_normal((P, 1, 3)).astype(np.float32),
        features_rest=(0.2 * rng.standard_normal((P, M - 1, 3))).astype(np.float32),
    )
    rot = raw["rotation"]
    act = dict(
        means3D=raw["xyz"],
        scales=np.exp(raw["scaling"]).astype(np.float32),
        rotations=(rot / np.sqrt((rot * rot).sum(1, keepdims=True))).astype(np.float32),
        opacities=(1.0 / (1.0 + np.exp(-raw["opacity"]))).astype(np.float32),
        shs=np.ascontiguousarray(np.concatenate([raw["features_dc"], raw["features_rest"]], axis=1)),
    )
    return dict(raw=raw, act=act, sh_degree=sh_degree, P=P, M=M)


def blender_frame(cam: SynthCamera, file_path: str) -> dict:
    """One `frames[]` entry of a NeRF-synthetic transforms_*.json for this camera: `transform_matrix` is camera-to-world in
    the OpenGL/Blender convention, i.e. the COLMAP camera-to-world with its y and z axes negated -- exactly what
    scene/dataset_readers.py:237-246 undoes when it loads the file."""
    w2c = np.asarray(cam.world_view_transform, np.float64).T
    c2w = np.linalg.inv(w2c)
    c2w[:3, 1:3] *= -1.0
    return {"file_path": file_path, "transform_matrix": c2w.tolist()}


def _write_points_ply(path: str, n_points: int, seed: int) -> None:
    """points in the layout of storePly (scene/dataset_readers.py:146-163): x y z nx ny nz (f4) red green blue (u1)"""
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(-1.0, 1.0, (n_points, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (n_points, 3)).astype(np.uint8)
    dt = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                   ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    v = np.zeros(n_points, dt)
    v["x"], v["y"], v["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    v["red"], v["green"], v["blue"] = rgb[:, 0], rgb[:, 1], rgb[:, 2]
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % n_points).encode())
        for n_, t_ in (("x", "float"), ("y", "float"), ("z", "float"), ("nx", "float"), ("ny", "float"), ("nz", "float"),
                       ("red", "uchar"), ("green", "uchar"), ("blue", "uchar")):
            f.write(f"property {t_} {n_}\n".encode())
        f.write(b"end_header\n")
        f.write(v.tobytes())


def _rotmat_to_qvec(R: np.ndarray) -> np.ndarray:
    """(w, x, y, z) of a rotation matrix; inverse of scene/colmap_loader.py:47-66 qvec2rotmat."""
    m = np.asarray(R, np.float64)
    K = np.array([[m[0, 0] - m[1, 1] - m[2, 2], 0, 0, 0],
                  [m[1, 0] + m[0, 1], m[1, 1] - m[0, 0] - m[2, 2], 0, 0],
                  [m[2, 0] + m[0, 2], m[2, 1] + m[1, 2], m[2, 2] - m[0, 0] - m[1, 1], 0],
                  [m[2, 1] - m[1, 2], m[0, 2] - m[2, 0], m[1, 0] - m[0, 1], m[0, 0] + m[1, 1] + m[2, 2]]]) / 3.0
    w, V = np.linalg.eigh(K)
    q = V[[3, 0, 1, 2], np.argmax(w)]
    return -q if q[0] < 0 else q


def write_colmap_dataset(path: str, views, n_points: int = 2000, seed: int = 0) -> None:
    """Write a COLMAP-layout dataset the reference's Scene loads unmodified (scene/dataset_readers.py:78-218 through the TEXT
    fallback of scene/colmap_loader.py:183-207,289-321): sparse/0/{cameras.txt, images.txt, points3D.ply} + images/r_XXX.png.
    `views`: list of (SynthCamera, image float32 [3,H,W] in [0,1]); one shared PINHOLE camera.  With `--eval` the loader holds
    out every 8th image (sorted by name) as the test set (dataset_readers.py:186-191).
    (This image's Pillow rejects `Image.fromarray(int8_array, "RGB")`, which the reference's Blender loader calls at
    dataset_readers.py:257, so the NeRF-synthetic layout of write_blender_dataset cannot be loaded by the unmodified reference here.)"""
    import os
    from PIL import Image
    os.makedirs(os.path.join(path, "sparse", "0"), exist_ok=True)
    os.makedirs(os.path.join(path, "images"), exist_ok=True)
    cam0 = views[0][0]
    W, H = cam0.image_width, cam0.image_height
    fx, fy = W / (2.0 * cam0.tanfovx), H / (2.0 * cam0.tanfovy)
    with open(os.path.join(path, "sparse", "0", "cameras.txt"), "w") as f:
        f.write("# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n")
        f.write(f"1 PINHOLE {W} {H} {fx!r} {fy!r} {W / 2.0!r} {H / 2.0!r}\n")
    with open(os.path.join(path, "sparse", "0", "images.txt"), "w") as f:
        f.write("# IMAGE_ID, QW, QX, QY, QZ, TX, TY, TZ, CAMERA_ID, NAME\n#   POINTS2D[] as (X, Y, POINT3D_ID)\n")
        for k, (cam, img) in enumerate(views):
            assert (cam.image_width, cam.image_height) == (W, H)
            name = f"r_{k:03d}.png"
            a = np.clip(np.asarray(img, np.float32), 0.0, 1.0)
            Image.fromarray(np.rint(a.transpose(1, 2, 0) * 255.0).astype(np.uint8), "RGB").save(os.path.join(path, "images", name))
            w2c = np.asarray(cam.world_view_transform, np.float64).T
            q, t = _rotmat_to_qvec(w2c[:3, :3]), w2c[:3, 3]
            f.write(f"{k + 1} {q[0]!r} {q[1]!r} {q[2]!r} {q[3]!r} {t[0]!r} {t[1]!r} {t[2]!r} 1 {name}\n\n".replace("np.float64(", "").replace(")", ""))
    _write_points_ply(os.path.join(path, "sparse", "0", "points3D.ply"), n_points, seed)


def write_blender_dataset(path: str, train, test, n_points: int = 2000, seed: int = 0) -> None:
    """Write a NeRF-synthetic ("Blender") dataset the reference's Scene loads unmodified (scene/dataset_readers.py:222-306):
    transforms_train.json / transforms_test.json (the loader REQUIRES both), RGBA PNGs, and a small points3d.ply so that the loader
    does not generate its 100 000 random points.  `train` / `test`: lists of (SynthCamera, image float32 [3,H,W] in [0,1]).
    All cameras must share FoVx (the format stores one `camera_angle_x` per file)."""
    import json
    import os
    from PIL import Image
    os.makedirs(path, exist_ok=True)
    for name, items in (("train", train), ("test", test)):
        os.makedirs(os.path.join(path, name), exist_ok=True)
        frames = []
        for k, (cam, img) in enumerate(items):
            rel = f"{name}/r_{k}"
            a = np.clip(np.asarray(img, np.float32), 0.0, 1.0)
            rgba = np.concatenate([np.rint(a.transpose(1, 2, 0) * 255.0).astype(np.uint8),
                                   np.full(a.shape[1:] + (1,), 255, np.uint8)], axis=2)
            Image.fromarray(rgba, "RGBA").save(os.path.join(path, rel + ".png"))
            frames.append(blender_frame(cam, rel))
        fovx = items[0][0].FoVx if items else math.radians(60.0)
        with open(os.path.join(path, f"transforms_{name}.json"), "w") as f:
            json.dump({"camera_angle_x": fovx, "frames": frames}, f)
    _write_points_ply(os.path.join(path, "points3d.ply"), n_points, seed)
