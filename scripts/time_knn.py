#!/usr/bin/env python
"""Time distCUDA2 three ways, alternating them: ours (lgr_knn_mean_dist3), the reference's extension (oracle/_ref/stock/simple_knn, in
its own process under the stock stack's import path) and the torch formulation this project used before (cdist on row chunks + topk,
restated below).  CUDA events around each call after a warm-up; median, p10 and p90 per implementation and size.

    python scripts/time_knn.py [--sizes 100000,1000000,3000000] [--iters 10] [--rounds 3] [--out FILE.json]

The torch formulation is O(P^2); it is skipped (reported "not measured") where one call is predicted, from its time at the smallest
size, to take more than a minute."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def torch_formulation(points):
    import torch
    P = points.shape[0]
    out = torch.empty(P, device=points.device, dtype=points.dtype)
    step = max(1, min(P, (1 << 26) // max(P, 1)))
    for s in range(0, P, step):
        d = torch.cdist(points[s:s + step], points)
        out[s:s + step] = (d.topk(4, dim=1, largest=False).values[:, 1:] ** 2).mean(dim=1)
    return out


def time_calls(fn, x, iters, warmup):
    import torch
    for _ in range(warmup):
        fn(x)
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn(x)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return ms


def ref_worker(path, iters, warmup):
    import torch
    from simple_knn._C import distCUDA2
    x = torch.from_numpy(np.load(path)).cuda()
    print("REFMS " + json.dumps(time_calls(distCUDA2, x, iters, warmup)))


def run_reference(x, iters, warmup):
    sys.path.insert(0, ROOT)
    from tests import scripts_harness as H
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "x.npy")
        np.save(p, x)
        out = H.run("stock", [os.path.abspath(__file__), "--ref-worker", p, str(iters), str(warmup)], cwd=d)
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("REFMS ")][-1]
    return json.loads(line[6:])


def stats(ms):
    if not ms:
        return "not measured"
    a = np.asarray(ms)
    return {"median_ms": float(np.median(a)), "p10_ms": float(np.percentile(a, 10)), "p90_ms": float(np.percentile(a, 90)), "n": len(ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,1000000,3000000")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--ref-worker", nargs=3, default=None)
    a = ap.parse_args()
    if a.ref_worker:
        ref_worker(a.ref_worker[0], int(a.ref_worker[1]), int(a.ref_worker[2]))
        return
    import torch
    assert torch.cuda.is_available(), "time_knn.py needs a GPU"
    sys.path.insert(0, ROOT)
    from lightgaussian_b200.knn import distCUDA2
    from lightgaussian_b200.synth import make_scene
    from tests.scripts_harness import stacks_available
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()
    have_ref = os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "stock", "simple_knn")) and stacks_available() is None
    result = {"card": card, "sizes": {}}
    torch_ms_per_p2 = None
    for P in [int(s) for s in a.sizes.split(",")]:
        x = make_scene(P, sh_degree=0, seed=P)["raw"]["xyz"]
        xt = torch.from_numpy(x).cuda()
        run_torch = torch_ms_per_p2 is None or torch_ms_per_p2 * P * P < 60_000.0
        t = {"ours": [], "reference": [], "torch": []}
        for _ in range(a.rounds):
            t["ours"] += time_calls(distCUDA2, xt, a.iters, a.warmup)
            if have_ref:
                t["reference"] += run_reference(x, a.iters, a.warmup)
            if run_torch:
                t["torch"] += time_calls(torch_formulation, xt, max(1, a.iters // 5), 1)
        if t["torch"]:
            torch_ms_per_p2 = float(np.median(t["torch"])) / (P * P)
        row = {k: stats(v) for k, v in t.items()}
        result["sizes"][P] = row
        print(json.dumps({"P": P, **row}), flush=True)
    print("card:", card)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
