"""distCUDA2 on the GPU (lightgaussian_b200/knn.py -> lgr_knn_mean_dist3, csrc/lgr_knn.cuh).  Every element is compared; "bit-identical"
means equal float32 bit patterns.  The reference's own extension (oracle/_ref/stock/simple_knn, staged by oracle/stage_reference.py) runs
in a subprocess under the stock stack's import path, never next to dropin/ on sys.path; those tests skip where it was not built."""
import os
import tempfile

import numpy as np
import pytest
import torch

from tests.knn_clouds import SHAPES, SIZES, cloud, mean_dist3_float64, sfm_like

pytestmark = pytest.mark.gpu

FLT_MAX = np.float32(np.finfo(np.float32).max)
REF_KNN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "stock", "simple_knn")


def ours(x: np.ndarray) -> np.ndarray:
    from lightgaussian_b200.knn import distCUDA2
    out = distCUDA2(torch.from_numpy(x).cuda())
    assert out.dtype == torch.float32 and out.shape == (x.shape[0],) and out.is_cuda
    return out.cpu().numpy()


def assert_bits_equal(got, want, what):
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    assert got.shape == want.shape, what
    bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, f"{what}: {bad.size} of {got.size} elements differ, first {bad[:5].tolist()}: {got[bad[:5]]} vs {want[bad[:5]]}"


def reference_available():
    return os.path.isdir(REF_KNN) and any(f.startswith("_C") and f.endswith(".so") for f in os.listdir(REF_KNN))


needs_reference = pytest.mark.skipif(not reference_available(), reason="oracle/_ref/stock/simple_knn (the reference's extension) is not built")


def reference(clouds: dict) -> dict:
    """the reference's distCUDA2 on each cloud, one subprocess for all of them"""
    from tests import scripts_harness as H
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.npz"), os.path.join(d, "out.npz")
        np.savez(src, **clouds)
        H.run("stock", [os.path.join(H.HELPERS, "ref_distcuda2.py"), src, dst], cwd=d)
        with np.load(dst) as f:
            out = {k: f[k] for k in f.files}
    # the stock stack must have run the reference's extension, not a drop-in shadowing it
    module = str(out.pop("__module__"))
    assert os.path.realpath(module).startswith(os.path.realpath(REF_KNN) + os.sep), module
    return out


@pytest.mark.parametrize("shape", SHAPES)
def test_bit_identical_to_oracle(shape):
    from oracle.knn_oracle import knn_mean_dist3
    for P in SIZES:
        x = cloud(shape, P, seed=P)
        assert_bits_equal(ours(x), knn_mean_dist3(x), f"{shape} P={P}")


def test_fewer_than_four_points():
    from oracle.knn_oracle import knn_mean_dist3
    assert ours(np.zeros((0, 3), np.float32)).shape == (0,)
    clouds = {f"p{P}": cloud("uniform", P, seed=P) for P in (1, 2, 3)}
    got = {k: ours(x) for k, x in clouds.items()}
    # the reference's FLT_MAX placeholders, summed (b0 + b1) + b2 and divided by 3
    assert np.all(np.isposinf(got["p1"])) and np.all(np.isposinf(got["p2"]))
    assert np.all(got["p3"] == FLT_MAX / np.float32(3.0))
    for k, x in clouds.items():
        assert_bits_equal(got[k], knn_mean_dist3(x), k)
    if reference_available():
        ref = reference(clouds)
        for k in clouds:
            assert_bits_equal(got[k], ref[k], f"{k} vs the reference's extension")


@needs_reference
def test_bit_identical_to_reference_on_shapes():
    clouds = {f"{s}_{P}": cloud(s, P, seed=P) for s in SHAPES for P in SIZES}
    ref = reference(clouds)
    for k, x in clouds.items():
        assert_bits_equal(ours(x), ref[k], k)


@needs_reference
def test_bit_identical_to_reference_at_scale():
    from lightgaussian_b200.synth import make_scene
    clouds = {f"scene_{P}": make_scene(P, sh_degree=0, seed=P)["raw"]["xyz"] for P in (1_000_000, 3_000_000)}
    clouds["sfm_1M"] = sfm_like(1_000_000, seed=11)
    ref = reference(clouds)
    for k, x in clouds.items():
        assert_bits_equal(ours(x), ref[k], k)


def test_against_float64_kdtree_at_1M():
    from lightgaussian_b200.synth import make_scene
    for name, x in (("scene", make_scene(1_000_000, sh_degree=0, seed=3)["raw"]["xyz"]), ("sfm", sfm_like(1_000_000, seed=4))):
        got = ours(x).astype(np.float64)
        want = mean_dist3_float64(x)
        err = np.abs(got - want)
        assert np.all(err <= 1e-6 * want), f"{name}: max rel err {np.max(err / np.maximum(want, 1e-300)):.3g}"


def test_input_handling():
    from lightgaussian_b200.knn import distCUDA2
    x = torch.from_numpy(sfm_like(100_000, seed=5)).cuda()
    a = distCUDA2(x)
    for _ in range(3):
        assert_bits_equal(distCUDA2(x).cpu().numpy(), a.cpu().numpy(), "repeat")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b = distCUDA2(x)
    torch.cuda.current_stream().wait_stream(s)
    assert_bits_equal(b.cpu().numpy(), a.cpu().numpy(), "non-default stream")
    wide = torch.cat([x, torch.rand(x.shape[0], 1, device="cuda")], dim=1)
    view = wide[:, :3]
    assert not view.is_contiguous()
    assert_bits_equal(distCUDA2(view).cpu().numpy(), a.cpu().numpy(), "column slice of [P,4]")
    with pytest.raises(RuntimeError):
        distCUDA2(x.cpu())
    with pytest.raises(RuntimeError):
        distCUDA2(x.double())


def _write_sfm_ply(path, xyz):
    """points3D.ply in the layout synth.write_colmap_dataset writes (storePly, scene/dataset_readers.py:146-163)"""
    dt = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                   ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    v = np.zeros(len(xyz), dt)
    v["x"], v["y"], v["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    v["red"] = 128
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % len(xyz)).encode())
        for n_ in ("x", "y", "z", "nx", "ny", "nz"):
            f.write(f"property float {n_}\n".encode())
        for n_ in ("red", "green", "blue"):
            f.write(f"property uchar {n_}\n".encode())
        f.write(b"end_header\n")
        f.write(v.tobytes())


@needs_reference
def test_scene_creation_scales_match_the_stock_stack():
    """Scene(dataset, GaussianModel(3)) through the unmodified reference code: create_from_pcd's initial _scaling, ours vs stock."""
    from tests import scripts_harness as H
    from lightgaussian_b200.synth import make_cameras, write_colmap_dataset
    reason = H.stacks_available()
    if reason:
        pytest.skip(reason)
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "data")
        rng = np.random.default_rng(0)
        views = [(c, rng.random((3, 48, 64)).astype(np.float32)) for c in make_cameras(4, 64, 48)]
        write_colmap_dataset(src, views, n_points=10)
        xyz = sfm_like(150_000, seed=6)
        _write_sfm_ply(os.path.join(src, "sparse", "0", "points3D.ply"), xyz)
        scal = {}
        for stack in ("ours", "stock"):
            model = os.path.join(d, f"model_{stack}")
            os.makedirs(model)
            out = os.path.join(d, f"scaling_{stack}.npy")
            run = H.run(stack, [os.path.join(H.HELPERS, "scene_scaling.py"), src, model, out])
            if stack == "stock":   # the reference's own extension, not a drop-in
                line = [ln for ln in run.stdout.splitlines() if ln.startswith("distCUDA2 from ")][-1]
                assert os.path.realpath(line[len("distCUDA2 from "):]).startswith(os.path.realpath(REF_KNN) + os.sep), line
            scal[stack] = np.load(out)
        assert scal["ours"].shape == (len(xyz), 3)
        assert_bits_equal(scal["ours"], scal["stock"], "_scaling after create_from_pcd")
