"""Time the view-parallel densification statistics at 3M Gaussians, 1080p, 8 ranks simulated on one GPU (every rank's exchange buffer
on this device, push layout): the sparse pack with statistics off and on, lgr_densify_stats_exchanged, and the all-gather path's two
kernels (encode, add views) without the NCCL all-gather itself.  CUDA events, alternating rounds, warm-up first; prints the card name
and power limit with the numbers.

    python scripts/time_densify_exchange.py [--rounds 7] [--iters 20]

On one GPU the pack's push stores to the 7 peer slots are local HBM stores, not NVLink: the pack numbers are the kernels' cost, not
the exchange's."""
import argparse
import ctypes as C
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lightgaussian_b200 import capi, densify  # noqa: E402
from lightgaussian_b200.model import GaussianParams, TorchCamera  # noqa: E402
from lightgaussian_b200.rasterizer import (GaussianRasterizationSettings, _exchange_tables, _forward_raw_native, _make_view,  # noqa: E402
                                           _raw_struct, _sparse_pack)
from lightgaussian_b200.synth import make_cameras, make_scene  # noqa: E402

P, W, H, WORLD = 3_000_000, 1920, 1080, 8


def settings(cam):
    t = TorchCamera(cam, "cuda")
    return GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, torch.zeros(3, device="cuda"), 1.0, t.world_view_transform,
                                         t.full_proj_transform, 3, t.camera_center, False, False, False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("GPU:", smi.stdout.strip() or torch.cuda.get_device_name(0))
    lib = capi.load()
    raw = make_scene(P, sh_degree=3, seed=0)["raw"]
    pc = GaussianParams(raw, 3, "cuda", requires_grad=False)
    del raw
    leaves = [p.detach() for p in pc.parameters()]
    cams = make_cameras(16, W, H)[:WORLD]
    slot = (int(lib.lgr_sparse_exchange_bytes_stats(P)) + 255) // 256 * 256
    bufs = [torch.zeros(WORLD * slot // 4, dtype=torch.float32, device="cuda") for _ in range(WORLD)]
    pack, ptrs = zip(*[_exchange_tables([[b.data_ptr() for b in bufs]], r, slot, True) for r in range(WORLD)])
    ws = torch.empty(int(lib.lgr_sparse_workspace_bytes(P)), dtype=torch.uint8, device="cuda")
    ranks = [type("Rank", (), dict(pack_tables=pack[r], ptr_tables=ptrs[r], rank=r, push=True, ws=ws))() for r in range(WORLD)]
    serial = 1
    gen = torch.Generator().manual_seed(1234)
    g2d, filt = [], []
    keep = None
    for v in range(WORLD):                 # every rank's view, packed with statistics once
        rs = settings(cams[v])
        with torch.no_grad():
            _, _, R, color, radii, geom, binning, img, _ = _forward_raw_native(False, rs, *leaves)
        dpix = torch.sign(color - torch.rand(3, H, W, generator=gen).cuda()) / float(3 * H * W)
        g = torch.empty((P, 3), device="cuda")
        _sparse_pack(ranks[v], 0, rs, R, dpix, *leaves, radii, geom, binning, img, g, serial=serial)
        g2d.append(g)
        filt.append((radii > 0).contiguous())
        if v == 0:
            keep = (rs, radii, geom)       # rank 0's blend-backward accumulators: the timed packs start from them
        else:
            del geom
        del binning, img
    rs0, radii0, geom0 = keep
    view, _keep = _make_view(torch.device("cuda"), rs0.bg, rs0.viewmatrix, rs0.projmatrix, rs0.campos, rs0.tanfovx, rs0.tanfovy, H, W, 1.0, 3,
                             False, False)
    params = _raw_struct(*leaves)
    stream = capi.current_stream_ptr(torch.device("cuda"))
    st = capi.LgrSparseStats(serial)
    g_tmp = torch.empty((P, 3), device="cuda")

    def pack_off():
        lib.lgr_backward_raw_sparse_pack_push(C.byref(view), P, 16, C.byref(params), radii0.data_ptr(), geom0.data_ptr(), ranks[0].pack_tables[0],
                                              WORLD, 0, ws.data_ptr(), g_tmp.data_ptr(), stream)

    def pack_on():
        lib.lgr_backward_raw_sparse_pack_push_ex(C.byref(view), P, 16, C.byref(params), radii0.data_ptr(), geom0.data_ptr(),
                                                 ranks[0].pack_tables[0], WORLD, 0, ws.data_ptr(), g_tmp.data_ptr(), C.byref(st), stream)

    accum, denom = torch.zeros((P, 1), device="cuda"), torch.zeros((P, 1), device="cuda")
    views = torch.empty((WORLD, P), device="cuda")

    def exchanged():   # rank 1's call: the stats-off packs above rewrite rank 0's slot, which only rank 0's call checks
        densify.stats_exchanged(ranks[1], 0, 1, serial, WORLD, g2d[1], filt[1], accum, denom)

    def encode():
        views[0].copy_(densify.stats_encode(g2d[0], filt[0]))

    def add_views():
        densify.stats_add_views(views, accum, denom)

    for v in range(WORLD):
        views[v] = densify.stats_encode(g2d[v], filt[v])
    fns = {"pack (stats off)": pack_off, "pack (stats on)": pack_on, "lgr_densify_stats_exchanged": exchanged,
           "lgr_densify_stats_encode": encode, "lgr_densify_stats_add_views": add_views}
    times = {k: [] for k in fns}
    for rnd in range(args.rounds + 1):     # round 0 is the warm-up
        order = list(fns) if rnd % 2 == 0 else list(reversed(list(fns)))
        for name in order:
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                fns[name]()
            b.record()
            torch.cuda.synchronize()
            if rnd:
                times[name].append(a.elapsed_time(b) / args.iters)
    assert int(densify.error_word(torch.device("cuda")).item()) == 0
    rows = [int(bufs[0][v * slot // 4 + 3:v * slot // 4 + 4].view(torch.int32).item()) for v in range(WORLD)]
    print(f"P = {P}, {W}x{H}, {WORLD} simulated ranks; rows per view {rows}; visible in view 0: {int(filt[0].sum())}")
    for name, t in times.items():
        t = sorted(t)
        print(f"{name}: median {t[len(t) // 2]:.4f} ms, min {t[0]:.4f} ms")


if __name__ == "__main__":
    main()
