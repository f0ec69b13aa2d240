"""GPU experiment: find the explicit operation order that reproduces, bit for bit, the torch operations of
GaussianModel.add_densification_stats / densify_and_split (scene/gaussian_model.py): torch.norm of a 2-vector, build_rotation, the
batched 3x3 . 3x1 bmm and log(exp(s) / (0.8*2)); and check that `empty(2S,3).normal_(0,1) * std + 0` draws what
torch.normal(mean=zeros, std=std) draws and leaves the CUDA generator in the same state.  Needs the staged reference tree
(oracle/_ref/stock/LightGaussian) for build_rotation and scripts/_build/libexp_densify.so (see scripts/exp_densify.cu)."""
import ctypes as C
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref", "stock", "LightGaussian"))
from utils.general_utils import build_rotation  # noqa: E402

lib = C.CDLL(os.path.join(ROOT, "scripts", "_build", "libexp_densify.so"))
vp, i32 = C.c_void_p, C.c_int
lib.run_norm2.argtypes = [vp, vp, i32, i32]
lib.run_rot.argtypes = [vp, vp, i32]
lib.run_bmm.argtypes = [vp, vp, vp, i32, i32]
lib.run_child_scale.argtypes = [vp, vp, i32, i32]
bits = lambda t: t.contiguous().view(torch.int32)  # noqa: E731
print(torch.cuda.get_device_name(0))

g = torch.Generator().manual_seed(0)
n = 3_000_000
# view-space gradients: magnitudes over many binades, both signs, exact zeros
grad = (torch.randn(n, 3, generator=g) * torch.exp(torch.randn(n, 3, generator=g) * 4 - 10)).cuda()
grad[::97, 0] = 0
mask = torch.rand(n, generator=g).cuda() > 0.3
ref = torch.norm(grad[mask, :2], dim=-1, keepdim=True)
sub = grad[mask].contiguous()
for v in range(3):
    y = torch.empty(sub.shape[0], device="cuda")
    lib.run_norm2(sub.data_ptr(), y.data_ptr(), sub.shape[0], v)
    print("norm2 variant", v, "mismatches", int((bits(y) != bits(ref[:, 0])).sum()), "of", sub.shape[0])

grads = (ref[:, 0] / torch.randint(1, 40, (ref.shape[0],), generator=g).float().cuda())[:, None]
clone_norm = torch.norm(grads, dim=-1)
print("norm of a one-element row: mismatches against sqrt(g*g)", int((bits(clone_norm) != bits(torch.sqrt(grads * grads)[:, 0])).sum()),
      "against |g|", int((bits(clone_norm) != bits(grads.abs()[:, 0])).sum()))

rot = torch.randn(n, 4, generator=g).cuda()
R = build_rotation(rot)
Rk = torch.empty(n, 9, device="cuda")
lib.run_rot(rot.data_ptr(), Rk.data_ptr(), n)
print("build_rotation mismatching rows", int((bits(Rk) != bits(R.reshape(n, 9))).any(1).sum()))

scal = (torch.randn(n, 3, generator=g) - 4).cuda()
samples = torch.normal(torch.zeros(n, 3, device="cuda"), torch.exp(scal))
for batch in (1, 2, 66, 4096, 8194, 100_000, n):
    ref = torch.bmm(R[:batch], samples[:batch].unsqueeze(-1)).squeeze(-1)
    res = []
    for v in range(9):
        y = torch.empty(batch, 3, device="cuda")
        lib.run_bmm(R.data_ptr(), samples.data_ptr(), y.data_ptr(), batch, v)
        res.append(int((bits(y) != bits(ref)).any(1).sum()))
    print("bmm batch", batch, "mismatching rows per variant", res)

ref = torch.log(torch.exp(scal) / (0.8 * 2))
for v in range(2):
    y = torch.empty_like(scal)
    lib.run_child_scale(scal.data_ptr(), y.data_ptr(), scal.numel(), v)
    print("child scaling variant", v, "mismatches", int((bits(y) != bits(ref)).sum()))

for S in (0, 1, 5, 1000, 123457):
    std = torch.exp(scal[:S]).repeat(2, 1)
    torch.manual_seed(11 + S)
    a = torch.normal(mean=torch.zeros((std.size(0), 3), device="cuda"), std=std)
    sa = torch.cuda.get_rng_state()
    torch.manual_seed(11 + S)
    b = torch.empty(2 * S, 3, device="cuda").normal_(0, 1) * std + 0.0
    sb = torch.cuda.get_rng_state()
    print("normal S", S, "sample mismatches", int((bits(a) != bits(b)).sum()), "generator state equal", bool(torch.equal(sa, sb)),
          "state moved", not torch.equal(sa, (torch.manual_seed(11 + S), torch.cuda.get_rng_state())[1]))
