"""2-GPU (NCCL) check of the view-parallel path on real renders; skipped on a machine with one GPU."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _setup(device):
    from lightgaussian_b200.model import GaussianParams, TorchCamera, pipeline_params
    from lightgaussian_b200.synth import make_scene, make_cameras
    scene = make_scene(20000, seed=5, scale_mult=1.5)
    pc = GaussianParams(scene["raw"], 3, device)
    cams = [TorchCamera(c, device) for c in make_cameras(6, 320, 240)]
    return pc, cams, pipeline_params(), torch.zeros(3, device=device)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    from lightgaussian_b200 import parallel
    from lightgaussian_b200.renderer import render, count_render
    parallel.init_from_env("nccl")
    dev = torch.device("cuda", rank)
    pc, cams, pipe, bg = _setup(dev)
    cnt, imp = parallel.sharded_prune_list(pc, cams, pipe, bg, count_render, rank, world)
    flat = parallel.FlatGrads(pc.parameters())
    pkg = render(cams[rank], pc, pipe, bg)
    pkg["render"].sum().backward()
    flat.allreduce(world)
    torch.cuda.synchronize()
    # the same step with the compact exchange fused into backward()
    parallel.enable_gradient_exchange(world)
    for p in pc.parameters():
        p.grad = None
    render(cams[rank], pc, pipe, bg)["render"].sum().backward()
    parallel.enable_gradient_exchange(1)
    fused = torch.cat([p.grad.reshape(-1) for p in pc.parameters()])
    torch.cuda.synchronize()
    torch.save(dict(cnt=cnt.cpu(), imp=imp.cpu(), flat=flat.flat.cpu(), fused=fused.cpu()), os.path.join(out, f"r{rank}.pt"))
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_results_equal_single_gpu(tmp_path):
    import torch.multiprocessing as mp
    from lightgaussian_b200 import parallel
    from lightgaussian_b200.renderer import render, count_render
    world, port = 2, _free_port()
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    dev = torch.device("cuda", 0)
    pc, cams, pipe, bg = _setup(dev)
    cnt1, imp1 = parallel.sharded_prune_list(pc, cams, pipe, bg, count_render, 0, 1)
    grads = []
    for r in range(world):
        for p in pc.parameters():
            p.grad = None
        render(cams[r], pc, pipe, bg)["render"].sum().backward()
        grads.append(torch.cat([p.grad.reshape(-1) for p in pc.parameters()]).cpu())
    both = [torch.load(os.path.join(tmp_path, f"r{r}.pt")) for r in range(world)]
    assert torch.equal(both[0]["fused"], both[1]["fused"])   # the exchanged gradients are bit-identical on every rank: replicas cannot drift
    for r in range(world):
        d = both[r]
        assert torch.equal(d["cnt"], cnt1.cpu())      # significance: bit-identical for any partition
        assert torch.equal(d["imp"], imp1.cpu())
        ref = grads[0] + grads[1]
        rel = (d["flat"] - ref).abs().max() / ref.abs().max()
        assert rel < 1e-3                               # backward atomics are order-dependent run to run
        rel2 = (d["fused"] - ref).abs().max() / ref.abs().max()
        assert rel2 < 1e-3                              # compact SH exchange == dense all-reduce
