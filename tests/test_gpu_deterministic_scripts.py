"""The reference's training scripts, UNMODIFIED, on the native stack with LGR_DETERMINISTIC=1, each run twice from the same work
directory (tests/scripts_harness.py): every tensor of the saved checkpoint (parameters, optimizer state), imp_score.npz and
point_cloud.ply must be byte-identical between the two runs.
  * prune_finetune.py with an importance prune at its first iteration;
  * train_densify_prune.py from the SfM cloud, with densify-and-prune events at 100 and 200 and the importance prune at 260;
  * distill_train.py --augmented_view (the strided degree-2 student)."""
import os

import numpy as np
import pytest

from tests import scripts_harness as sh

pytestmark = pytest.mark.gpu

ITER0 = 30000
STEPS = 60
PORT = 6300


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    reason = sh.stacks_available()
    if reason:
        pytest.skip(reason)
    base = str(tmp_path_factory.mktemp("lgdet"))
    return sh.build_workdir(base, iteration=ITER0)


def _run_twice(argv_of):
    """argv_of(k) -> (argv, output directory, trace path); runs run k = 0, 1 with LGR_DETERMINISTIC=1; returns the directories and the
    traces of the library calls"""
    old = os.environ.get("LGR_DETERMINISTIC")
    os.environ["LGR_DETERMINISTIC"] = "1"
    try:
        outs, traces = [], []
        for k in range(2):
            a, out, trace = argv_of(k)
            sh.run("ours", a, trace=trace)
            outs.append(out)
            traces.append(sh.read_trace(trace))
        return outs, traces
    finally:
        if old is None:
            os.environ.pop("LGR_DETERMINISTIC", None)
        else:
            os.environ["LGR_DETERMINISTIC"] = old


def _same_object(a, b, where):
    import torch
    if isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape, where
        assert torch.equal(a.detach().cpu().reshape(-1).view(torch.uint8), b.detach().cpu().reshape(-1).view(torch.uint8)), where
    elif isinstance(a, dict):
        assert sorted(a, key=str) == sorted(b, key=str), where
        for k in a:
            _same_object(a[k], b[k], f"{where}/{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _same_object(x, y, f"{where}[{i}]")
    else:
        assert a == b, where


def _compare_outputs(d0, d1, need):
    """every checkpoint (tensor by tensor), every .npz (array by array) and every .ply (byte by byte) under the two output directories"""
    import torch

    def files(d):
        out = []
        for root, _, names in os.walk(d):
            out += [os.path.relpath(os.path.join(root, n), d) for n in names if n.endswith((".pth", ".npz", ".ply"))]
        return sorted(out)
    f0, f1 = files(d0), files(d1)
    assert f0 == f1, (f0, f1)
    for suffix in need:
        assert any(f.endswith(suffix) for f in f0), (suffix, f0)
    for f in f0:
        a, b = os.path.join(d0, f), os.path.join(d1, f)
        if f.endswith(".pth"):
            _same_object(torch.load(a, weights_only=False, map_location="cpu"), torch.load(b, weights_only=False, map_location="cpu"), f)
        elif f.endswith(".npz"):
            za, zb = np.load(a, allow_pickle=True), np.load(b, allow_pickle=True)
            assert sorted(za.files) == sorted(zb.files), f
            for k in za.files:
                assert za[k].dtype == zb[k].dtype and np.array_equal(za[k], zb[k]), (f, k)
        else:
            with open(a, "rb") as fa, open(b, "rb") as fb:
                assert fa.read() == fb.read(), f
    print(f"\n{len(f0)} files byte-identical: {f0}")


def test_prune_finetune_twice_bit_identical(work):
    last = ITER0 + STEPS

    def argv(k):
        out = os.path.join(work["base"], f"pf_det{k}")
        return (["prune_finetune.py", "-s", work["data"], "-m", out, "--eval", "-r", "1", "--port", str(PORT + k),
                 "--start_checkpoint", work["ckpt"], "--iterations", str(last), "--prune_percent", "0.66", "--prune_type", "v_important_score",
                 "--prune_decay", "1", "--v_pow", "0.1", "--position_lr_max_steps", str(last), "--prune_iterations", str(ITER0 + 1),
                 "--test_iterations", "999999", "--save_iterations", str(last), "--checkpoint_iterations", str(last)], out, out + ".trace.json")
    (d0, d1), _ = _run_twice(argv)
    _compare_outputs(d0, d1, [f"chkpnt{last}.pth", "imp_score.npz", "point_cloud.ply"])


def test_distill_train_augmented_view_twice_bit_identical(work):
    last = ITER0 + STEPS

    def argv(k):
        out = os.path.join(work["base"], f"dt_det{k}")
        return (["distill_train.py", "-s", work["data"], "-m", out, "--eval", "-r", "1", "--port", str(PORT + 10 + k),
                 "--start_checkpoint", work["ckpt"], "--teacher_model", work["ckpt"], "--iterations", str(last), "--new_max_sh", "2",
                 "--position_lr_max_steps", str(last), "--enable_covariance", "--augmented_view",
                 "--test_iterations", "999999", "--save_iterations", str(last), "--checkpoint_iterations", str(last)], out, out + ".trace.json")
    (d0, d1), _ = _run_twice(argv)
    _compare_outputs(d0, d1, [f"chkpnt{last}.pth", "imp_score.npz", "point_cloud.ply"])


def test_train_densify_prune_twice_bit_identical(work):
    from lightgaussian_b200.synth import make_cameras, make_scene, write_colmap_dataset
    scene = make_scene(20000, sh_degree=3, seed=5, scale_mult=1.5)
    cams = make_cameras(24, 320, 240)
    data = os.path.join(work["base"], "tdp_data")
    write_colmap_dataset(data, list(zip(cams, sh.render_ground_truth(scene["raw"], cams))), n_points=20000)
    last = 300

    def argv(k):
        out = os.path.join(work["base"], f"tdp_det{k}")
        return (["train_densify_prune.py", "-s", data, "-m", out, "--eval", "-r", "1", "--port", str(PORT + 20 + k),
                 "--iterations", str(last), "--densify_from_iter", "50", "--densification_interval", "100",
                 "--densify_until_iter", "250", "--opacity_reset_interval", "3000", "--prune_iterations", "260",
                 "--position_lr_max_steps", str(last), "--test_iterations", "999999", "--save_iterations", str(last),
                 "--checkpoint_iterations", str(last)], out, out + ".trace.json")
    (d0, d1), traces = _run_twice(argv)
    assert all(t.get("densify_native", 0) == 2 for t in traces), traces   # densify-and-prune at iterations 100 and 200
    _compare_outputs(d0, d1, [f"chkpnt{last}.pth", "point_cloud.ply"])
