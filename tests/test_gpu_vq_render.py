"""Rendering a VecTree-compressed model in place (lightgaussian_b200/vqresident.py, lgr_forward_vq).

The oracle is the existing fused render of the same model loaded the way GaussianModel.load_vq loads it (dense float32 leaves):
images, radii, visibility and the significance outputs must be torch.equal.  Fixtures are written by our Quantization (the
reference's writer) or, for what the writer cannot produce (vq_ratio 0, float32 attributes, P = 0), directly in the file format.
"""
import ctypes as C
import json
import math
import os
import shutil
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import scripts_harness as sh

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ply_table(raw, degree):
    """read_ply_data's [P, 6+D+8] table: xyz, normals (0), f_dc, f_rest channel-major, opacity, scale, rot"""
    P = raw["xyz"].shape[0]
    rest = raw["features_rest"][:, :(degree + 1) ** 2 - 1, :]
    return np.concatenate([raw["xyz"], np.zeros((P, 3), np.float32), raw["features_dc"].reshape(P, 3),
                           rest.transpose(0, 2, 1).reshape(P, 3 * rest.shape[1]), raw["opacity"], raw["scaling"], raw["rotation"]], axis=1).astype(np.float32)


def _write_direct(model_dir, table, D, nonvq_mask, codebook, idx, dtype):
    """extreme_saving/ in the writer's format (vectree/vectree.py:107-155), for inputs the writer cannot produce"""
    ex = os.path.join(model_dir, "extreme_saving")
    os.makedirs(ex, exist_ok=True)
    P, K = table.shape[0], codebook.shape[0]
    bits = int(math.log2(K))
    np.savez_compressed(os.path.join(ex, "metadata.npz"),
                        metadata=dict(input_pc_num=P, input_pc_dim=table.shape[1], codebook_size=K, codebook_dim=D))
    bitmat = ((idx.astype(np.int64)[:, None] >> np.arange(bits - 1, -1, -1)) & 1).astype(np.uint8)
    np.savez_compressed(os.path.join(ex, "vq_indexs.npz"), np.packbits(bitmat.reshape(-1)))
    np.savez_compressed(os.path.join(ex, "codebook.npz"), codebook.astype(np.float16))
    np.savez_compressed(os.path.join(ex, "non_vq_mask.npz"), np.packbits(nonvq_mask.astype(np.uint8)))
    np.savez_compressed(os.path.join(ex, "non_vq_feats.npz"), table[nonvq_mask, 6:6 + D].astype(dtype))
    np.savez_compressed(os.path.join(ex, "other_attribute.npz"), table[:, -8:].astype(dtype))
    np.savez_compressed(os.path.join(ex, "xyz.npz"), table[:, 0:3])


def make_model(model_dir, P, degree=3, vq_ratio=0.6, half=True, seed=0, codebook_size=256, writer=None):
    """A model directory with extreme_saving/.  writer None: our Quantization when it can write the case, else direct."""
    from lightgaussian_b200.synth import make_scene
    raw = make_scene(max(P, 1), sh_degree=3, seed=seed)["raw"]
    raw = {k: v[:P] for k, v in raw.items()}
    table = _ply_table(raw, degree)
    D = 3 * (degree + 1) ** 2
    if writer is None:
        writer = "quantization" if (P > 0 and 0 < vq_ratio and half) else "direct"
    if writer == "quantization":
        from lightgaussian_b200.vectree import Quantization
        imp = np.random.default_rng(seed + 1).random(P)
        torch.manual_seed(seed)
        q = Quantization(table, importance=imp, sh_degree=degree, save_path=model_dir, codebook_size=codebook_size, iteration_num=3,
                         vq_ratio=vq_ratio, vq_way="half", device=DEV, VQ_CHUNK=8000)
        q.quantize()
    else:
        rng = np.random.default_rng(seed + 2)
        nonvq = np.zeros(P, bool)
        nonvq[rng.permutation(P)[:int(P * (1 - vq_ratio))]] = True
        codebook = (0.3 * rng.standard_normal((codebook_size, D))).astype(np.float16)
        idx = rng.integers(0, codebook_size, int((~nonvq).sum()))
        _write_direct(model_dir, table, D, nonvq, codebook, idx, np.float16 if half else np.float32)
    return model_dir


class ResidentModel:
    """What render() needs from a GaussianModel whose leaves are deferred: _xyz, the store and the SH degrees."""

    def __init__(self, store, active=None):
        self._vq_resident = store
        self._xyz = store.xyz
        self.max_sh_degree = int(round(math.sqrt(store.D // 3))) - 1
        self.active_sh_degree = self.max_sh_degree if active is None else active

    @property
    def get_xyz(self):
        return self._xyz


def dense_model(store, active):
    from lightgaussian_b200.model import GaussianParams
    leaves = store.materialize()
    pc = GaussianParams.__new__(GaussianParams)
    for n, t in leaves.items():
        setattr(pc, n, t)
    pc.max_sh_degree, pc.active_sh_degree = store.max_sh_degree, active
    return pc


def cameras(W, H):
    from lightgaussian_b200.model import TorchCamera
    from lightgaussian_b200.synth import camera_from_pose, make_cameras
    cams = [TorchCamera(c) for c in make_cameras(2, W, H)]
    culled = TorchCamera(camera_from_pose(np.eye(3), np.array([0.0, 0.0, -5.0]), W, H, math.radians(60.0)))
    return cams, culled


def compare(store, cams, active, scaling_modifier=1.0, bg=(0.0, 0.0, 0.0)):
    from lightgaussian_b200 import trace
    from lightgaussian_b200.model import pipeline_params
    from lightgaussian_b200.renderer import count_render, render
    pipe = pipeline_params()
    bgt = torch.tensor(bg, dtype=torch.float32, device=DEV)
    res, den = ResidentModel(store, active), dense_model(store, active)
    with torch.no_grad():
        for cam in cams:
            for fn in (render, count_render):
                before = trace.counters.get("render_vq_resident", 0)
                a = fn(cam, res, pipe, bgt, scaling_modifier)
                assert trace.counters.get("render_vq_resident", 0) == before + 1
                b = fn(cam, den, pipe, bgt, scaling_modifier)
                keys = ["render", "radii", "visibility_filter"] + (["gaussians_count", "important_score"] if fn is count_render else [])
                for k in keys:
                    assert torch.equal(a[k], b[k]), (k, fn.__name__)
    return res


CASES = [  # P, degree, vq_ratio, half
    (0, 3, 0.6, True), (1, 3, 0.6, True), (31, 2, 0.6, True), (32, 3, 1.0, True), (33, 2, 0.0, True), (257, 3, 0.6, False),
    (4097, 2, 0.6, True), (4097, 3, 0.0, False), (100_000, 3, 0.6, True), (100_000, 2, 1.0, True), (100_000, 2, 0.6, False),
]


@pytest.mark.parametrize("P,degree,vq_ratio,half", CASES)
def test_resident_render_equals_dense_leaves(tmp_path, P, degree, vq_ratio, half):
    from lightgaussian_b200.vqresident import ResidentVQ
    make_model(str(tmp_path), P, degree, vq_ratio, half, seed=P % 97)
    store = ResidentVQ.load(str(tmp_path), degree, DEV)
    assert store.Dp == (32 if degree == 2 else 48)
    assert (store.attr.dtype == torch.float16) == half
    for W, H in ((1, 1), (17, 5), (320, 240)):
        cams, culled = cameras(W, H)
        compare(store, cams + [culled], degree)
    cams, culled = cameras(160, 120)
    compare(store, cams, degree, scaling_modifier=0.7, bg=(1.0, 0.5, 0.25))
    for active in range(degree):
        compare(store, cams, active)


def test_resident_render_at_3m_and_1080p(tmp_path):
    """3M Gaussians, degree 3, the reference's 0.6 / half, 1080p, with the writer's default codebook size"""
    from lightgaussian_b200.vqresident import ResidentVQ
    make_model(str(tmp_path), 3_000_000, 3, 0.6, True, seed=3, codebook_size=8192)
    store = ResidentVQ.load(str(tmp_path), 3, DEV)
    cams, culled = cameras(1920, 1080)
    compare(store, cams + [culled], 3)


def test_memory_of_a_resident_load_and_frame(tmp_path):
    """3M / degree 3 / 0.6 / half: the store is what the arrays' shapes say, no dense table is built while loading, a loaded model
    holds less than the dense leaves by at least their difference, and load plus one 1080p frame peaks below the dense path.  (The
    frame's own buffers, about 1.2 GB here, are the same on both paths, so the peak difference is smaller than the leaves.)"""
    from lightgaussian_b200.model import pipeline_params
    from lightgaussian_b200.renderer import render
    from lightgaussian_b200.vqresident import ResidentVQ
    P = 3_000_000
    make_model(str(tmp_path), P, 3, 0.6, True, seed=4, codebook_size=8192)
    n_nonvq = int(P * 0.4)
    expected = P * 3 * 4 + P * 8 * 2 + P * 4 + n_nonvq * 48 * 2 + 8192 * 48 * 2
    cam = cameras(1920, 1080)[0][0]
    bg = torch.zeros(3, device=DEV)
    peaks = {}
    for path in ("resident", "dense"):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        with torch.no_grad():
            store = ResidentVQ.load(str(tmp_path), 3, DEV)
            if path == "resident":
                torch.cuda.synchronize()
                held, load_peak = torch.cuda.memory_allocated() - base, torch.cuda.max_memory_allocated() - base
                assert store.nbytes() <= 1.05 * expected
                assert held <= 1.05 * expected, (held, expected)
                assert load_peak <= 1.25 * expected, (load_peak, expected)
                model = ResidentModel(store)
            else:
                dense_held = None
                del store
                # the reference-shaped load alone: load_vqgaussian's table, then the six leaves
                shell = SimpleNamespace(path=str(tmp_path), max_sh_degree=3, xyz=torch.empty(0, device=DEV))
                leaves = ResidentVQ.materialize(shell)
                model = dense_model(SimpleNamespace(materialize=lambda: leaves, max_sh_degree=3), 3)
                del leaves
                torch.cuda.synchronize()
                dense_held = torch.cuda.memory_allocated() - base
            render(cam, model, pipeline_params(), bg)
        torch.cuda.synchronize()
        peaks[path] = torch.cuda.max_memory_allocated() - base
        del model
        store = None
    leaves = P * (3 + 3 + 45 + 1 + 3 + 4) * 4
    print(f"peak over load + one 1080p frame: resident {peaks['resident'] / 2**20:.0f} MiB, dense {peaks['dense'] / 2**20:.0f} MiB; "
          f"store {expected / 2**20:.0f} MiB, dense leaves {leaves / 2**20:.0f} MiB")
    assert dense_held >= leaves and dense_held - held >= leaves - 1.05 * expected, (dense_held, held)
    assert peaks["resident"] < peaks["dense"], peaks


def test_input_checks_raise_before_any_launch(tmp_path):
    from lightgaussian_b200 import capi
    from lightgaussian_b200.rasterizer import GaussianRasterizationSettings, forward_vq_native
    from lightgaussian_b200.vqresident import ResidentVQ
    d = make_model(str(tmp_path / "ok"), 257, 3, 0.6, True, seed=1)
    with pytest.raises(ValueError, match="degree"):
        ResidentVQ.load(d, 2, DEV)
    bad = str(tmp_path / "f32cb")
    shutil.copytree(d, bad)
    cb = np.load(os.path.join(bad, "extreme_saving", "codebook.npz"))["arr_0"]
    np.savez_compressed(os.path.join(bad, "extreme_saving", "codebook.npz"), cb.astype(np.float32))
    with pytest.raises(ValueError, match="codebook"):
        ResidentVQ.load(bad, 3, DEV)
    bad = str(tmp_path / "trunc")
    shutil.copytree(d, bad)
    idx = np.load(os.path.join(bad, "extreme_saving", "vq_indexs.npz"))["arr_0"]
    np.savez_compressed(os.path.join(bad, "extreme_saving", "vq_indexs.npz"), idx[:-2])
    launches = capi.launch_count()
    with pytest.raises(ValueError, match="vq_indexs"):
        ResidentVQ.load(bad, 3, DEV)
    assert capi.launch_count() == launches
    # CPU arrays handed to the C entry point: refused by the binding and by lgr_forward_vq itself, before any launch
    store = ResidentVQ.load(d, 3, DEV)
    cam = cameras(32, 32)[0][0]
    rs = GaussianRasterizationSettings(32, 32, math.tan(cam.FoVx / 2), math.tan(cam.FoVy / 2), torch.zeros(3, device=DEV), 1.0,
                                       cam.world_view_transform, cam.full_proj_transform, 3, cam.camera_center, False, False, False)
    cpu = SimpleNamespace(**{k: getattr(store, k).cpu() for k in ("attr", "slot", "codebook", "nonvq")},
                          P=store.P, D=store.D, Dp=store.Dp, K=store.K)
    launches = capi.launch_count()
    with pytest.raises(RuntimeError):
        forward_vq_native(False, rs, store.xyz, cpu)
    lib = capi.load()
    params = capi.LgrVqResidentParams(store.xyz.data_ptr(), cpu.attr.data_ptr(), cpu.slot.data_ptr(), cpu.codebook.data_ptr(),
                                      cpu.nonvq.data_ptr(), 1, 1, store.D, store.Dp, store.K)
    out = torch.empty(3, 32, 32, device=DEV)
    radii = torch.empty(store.P, dtype=torch.int32, device=DEV)
    nr = C.c_int32(0)
    st = lib.lgr_forward_vq(None, store.P, C.byref(params), capi.ALLOC_CB, None, capi.ALLOC_CB, None, capi.ALLOC_CB, None,
                            out.data_ptr(), None, None, radii.data_ptr(), C.byref(nr), None)
    assert st != capi.LGR_OK and b"device memory" in lib.lgr_last_error()
    assert capi.launch_count() == launches


# ---- the reference's GaussianModel and scripts ----
@pytest.fixture(scope="module")
def stacks():
    reason = sh.stacks_available()
    if reason:
        pytest.skip(reason)


def test_materialised_leaves_and_gradients_match_the_reference_load_vq(tmp_path, stacks):
    """tests/helpers/vq_load_compare.py, under our stack: the patched load_vq against the class's own, on the same files"""
    make_model(str(tmp_path), 4097, 3, 0.6, True, seed=7)
    out = str(tmp_path / "result.json")
    sh.run("ours", [os.path.join(sh.HELPERS, "vq_load_compare.py"), str(tmp_path), out])
    res = json.load(open(out))
    assert res["patched"] and res["deferred_before_read"], res
    assert res["leaves_equal"] == ["_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity"], res
    for k in ("grads_equal", "override_color_equal", "cov3D_python_equal", "capture_equal"):
        assert res[k], (k, res)
    assert res["trace"].get("vq_materialize", 0) >= 1, res


def test_render_scripts_run_unmodified_with_load_vq(tmp_path, stacks):
    """render_video.py --load_vq on the stock stack and on ours writes byte-identical PNG frames; ours renders in place"""
    from lightgaussian_b200.synth import make_cameras, write_colmap_dataset
    W, H = 160, 120
    cams = make_cameras(12, W, H)
    data = str(tmp_path / "data")
    write_colmap_dataset(data, [(c, np.zeros((3, H, W), np.float32)) for c in cams])
    src = make_model(str(tmp_path / "model_src"), 20000, 3, 0.6, True, seed=9)
    os.makedirs(os.path.join(src, "point_cloud", "iteration_30000"))
    frames = {}
    for stack, script in (("stock", "render_video.py"), ("ours", "render_video.py"), ("ours", "render.py")):
        model = str(tmp_path / f"m_{stack}_{script[:-3]}")
        shutil.copytree(src, model)
        with open(os.path.join(model, "cfg_args"), "w") as f:
            f.write(f"Namespace(sh_degree=3, source_path={data!r}, model_path={model!r}, images='images', resolution=-1, "
                    f"white_background=False, data_device='cuda', eval=False)")
        trace = str(tmp_path / f"{stack}_{script}.trace.json")
        sh.run(stack, [script, "-m", model, "--skip_test", "--quiet", "--load_vq"], trace=trace)
        rdir = os.path.join(model, "train", "ours_30000", "renders")
        names = sorted(os.listdir(rdir))
        assert len(names) == len(cams)
        frames[(stack, script)] = [open(os.path.join(rdir, n), "rb").read() for n in names]
        if stack == "ours":
            tr = sh.read_trace(trace)
            assert tr.get("render_vq_resident", 0) >= len(names) and tr.get("vq_materialize", 0) == 0, tr
    for key in (("ours", "render_video.py"), ("ours", "render.py")):
        assert frames[key] == frames[("stock", "render_video.py")], key
