"""GPU parity of the VecTree row (N4): lgr_vq_assign / lgr_vq_ema_update / gather / pack / unpack through
lightgaussian_b200.vectree, against the float64 oracle (oracle/vq_oracle.py), the golden produced by the reference's own vectree
modules (tests/golden/pyref_vq.npz) and, at the reference's full size (80 000 x 8192 x 27), the reference's torch formulation.
Tolerances: code indices identical except where two codes are within float rounding of each other (checked in float64); EMA state
1e-4 relative (atomics / summation order); codec and file payloads bit-exact."""
import os

import numpy as np
import pytest
import torch

from lightgaussian_b200 import vectree as vt
from oracle import vq_oracle as vo

pytestmark = pytest.mark.gpu
G = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pyref_vq.npz")))
G["feats_sh"] = G["full_feats"][:, 6:33]   # the VQ'd SH columns of the full feature rows (stored once)
N, D, K, CHUNK, ITERS, KEXP = (int(v) for v in G["cfg"])


def _ties_only(x, embed, ours, ref):
    """True when every disagreement is a numerical tie: both codes equally near in float64 up to fp32 rounding of the expansion"""
    bad = np.where(ours != ref)[0]
    if len(bad) == 0:
        return True
    x64, e64 = x[bad].astype(np.float64), embed.astype(np.float64)
    da = ((x64 - e64[ours[bad]]) ** 2).sum(1)
    db = ((x64 - e64[ref[bad]]) ** 2).sum(1)
    tol = 2e-6 * ((x64 ** 2).sum(1) + (e64[ours[bad]] ** 2).sum(1)) + 1e-7
    return bool(np.all(np.abs(da - db) <= tol))


@pytest.mark.parametrize("n,d,K_", [(1, 27, 64), (257, 27, 8192), (5000, 48, 512), (3000, 3, 7), (999, 64, 100), (70000, 27, 300)])
def test_assign_matches_oracle(n, d, K_):
    rng = np.random.default_rng(n + d)
    x = rng.standard_normal((n, d)).astype(np.float32)
    e = rng.standard_normal((K_, d)).astype(np.float32) * 1.5
    idx = vt.vq_assign(torch.from_numpy(x).cuda(), torch.from_numpy(e).cuda()).cpu().numpy()
    ref, _ = vo.assign(x, e)
    assert idx.min() >= 0 and idx.max() < K_
    assert _ties_only(x, e, idx, ref)
    assert (idx != ref).mean() < 1e-3


def test_duplicate_codes_resolve_to_the_smallest_index():
    x = torch.randn(100, 27).cuda()
    e = torch.randn(10, 27).cuda()
    e = torch.cat([e, e, e], 0)
    idx = vt.vq_assign(x, e)
    assert int(idx.max()) < 10


def test_kmeans_iterations_follow_the_reference_golden():
    torch.manual_seed(0)
    model = vt.VectorQuantize(dim=D, codebook_size=K, decay=0.8, commitment_weight=1.0, use_cosine_sim=False, threshold_ema_dead_code=0)
    np.testing.assert_array_equal(model._codebook.embed.numpy(), G["embed_init"])            # same RNG consumption as vq.py:25-28
    model = model.cuda().train()
    cb = model._codebook
    for it in range(ITERS):
        sel = G[f"it{it}_indexes"]
        x, w = torch.from_numpy(G["feats_sh"][sel]).cuda(), torch.from_numpy(G["imp"][sel]).cuda()
        before = cb.embed[0].cpu().numpy().copy()
        quantize, ind, loss = model(x.unsqueeze(0), weight=w.reshape(1, -1, 1))
        assert quantize.shape == (1, CHUNK, D) and ind.shape == (1, CHUNK) and ind.dtype == torch.int64 and loss.shape == (1,)
        ours = ind[0].cpu().numpy()
        assert _ties_only(G["feats_sh"][sel], before, ours, G[f"it{it}_ind"])
        if np.array_equal(ours, G[f"it{it}_ind"]):
            np.testing.assert_allclose(cb.cluster_size.cpu().numpy(), G[f"it{it}_cluster_size"], rtol=1e-4, atol=1e-4)
            np.testing.assert_allclose(cb.embed.cpu().numpy(), G[f"it{it}_embed_after_ema"], rtol=1e-4, atol=2e-5)
            assert abs(float(loss) - float(G[f"it{it}_loss"][0])) <= 1e-5 * float(G[f"it{it}_loss"][0])
            if it == 0:
                np.testing.assert_allclose(quantize[0].cpu().numpy(), G["it0_quantize"], rtol=0, atol=1e-6)
        cb.embed.copy_(torch.from_numpy(G[f"it{it}_embed_after_replace"]).cuda())          # continue from the reference's state
        cb.cluster_size.copy_(torch.from_numpy(G[f"it{it}_cluster_size"]).cuda())


def test_codec_bit_exact_and_round_trip():
    idx = torch.from_numpy(G["codec_idx"]).cuda()
    packed = vt.pack_indices(idx, 13)
    np.testing.assert_array_equal(packed.cpu().numpy(), G["codec_packed"])
    np.testing.assert_array_equal(vt.unpack_indices(packed, idx.numel(), 13).cpu().numpy(), G["codec_idx"])
    rng = np.random.default_rng(1)
    for bits, n in [(1, 1), (1, 77), (3, 1000), (8, 513), (13, 4097), (16, 12345), (20, 99)]:
        v = rng.integers(0, 2 ** bits, n)
        p = vt.pack_indices(torch.from_numpy(v).cuda(), bits)
        np.testing.assert_array_equal(p.cpu().numpy(), vo.pack_indices(v, bits))
        np.testing.assert_array_equal(vt.unpack_indices(p, n, bits).cpu().numpy(), v)


def test_files_and_dequantize_match_the_reference(tmp_path):
    q = vt.Quantization(G["full_feats"], importance=G["imp"], sh_degree=2, save_path=str(tmp_path), codebook_size=K, iteration_num=0,
                        vq_ratio=0.6)
    q.select()
    np.testing.assert_array_equal(q.non_vq_mask.numpy(), G["non_vq_mask"])
    q.model_vq._codebook.embed.copy_(torch.from_numpy(G[f"it{ITERS - 1}_embed_after_replace"]).cuda())
    all_feat, all_indice = q.fully_vq_reformat()
    ours_idx = all_indice.cpu().numpy()
    assert _ties_only(G["feats_sh"], G[f"it{ITERS - 1}_embed_after_replace"][0], ours_idx, G["all_indice"])
    ex = os.path.join(str(tmp_path), "extreme_saving")
    same = np.array_equal(ours_idx, G["all_indice"])
    for name in ["codebook", "non_vq_mask", "non_vq_feats", "other_attribute", "xyz"] + (["vq_indexs"] if same else []):
        got = np.load(os.path.join(ex, name + ".npz"))["arr_0"]
        assert got.dtype == G[f"file_{name}"].dtype, name
        np.testing.assert_array_equal(got, G[f"file_{name}"], err_msg=name)
    meta = np.load(os.path.join(ex, "metadata.npz"), allow_pickle=True)["metadata"].item()
    assert [meta[k] for k in ("input_pc_num", "input_pc_dim", "codebook_size", "codebook_dim")] == [int(v) for v in G["file_metadata"]]
    if same:
        np.testing.assert_array_equal(all_feat.cpu().numpy(), G["all_feat"])
        np.testing.assert_array_equal(q.dequantize().cpu().numpy(), G["dequantized"])
    files = {n: np.load(os.path.join(ex, n + ".npz"))["arr_0"] for n in ["vq_indexs", "codebook", "non_vq_mask", "non_vq_feats", "other_attribute", "xyz"]}
    np.testing.assert_array_equal(q.dequantize().cpu().numpy(), vo.dequantize(files, G["file_metadata"]))


def test_training_reduces_the_weighted_error():
    rng = np.random.default_rng(3)
    centers = rng.standard_normal((200, 27)).astype(np.float32) * 2
    feats = centers[rng.integers(0, 200, 50000)] + 0.1 * rng.standard_normal((50000, 27)).astype(np.float32)
    full = np.zeros((50000, 6 + 27 + 8), np.float32)
    full[:, 6:33] = feats
    imp = rng.random(50000).astype(np.float32)
    torch.manual_seed(1)
    q = vt.Quantization(full, importance=imp, sh_degree=2, save_path=None, codebook_size=256, iteration_num=30, vq_ratio=0.6, VQ_CHUNK=8192)
    q.select()

    def err():
        feat, _ = q.calc_vector_quantized_feature()
        m = q.vq_mask.cuda()
        return float((((feat - q.feats) ** 2).sum(1) * m).sum() / m.sum())
    e0 = err()
    q.train_codebook()
    e1 = err()
    assert e1 < 0.3 * e0, (e0, e1)                        # measured: 0.13 after 30 iterations


def _torch_reference_iteration(x, w, embed, cluster_size, decay=0.8, eps=1e-5):
    """vq.py:262-300 restated with the same torch ops (cdist, argmax, one_hot, einsum) for the full-size comparison"""
    Kc = embed.shape[0]
    wn = (w * w.numel() / w.sum()).reshape(1, -1, 1)
    flat = x[None]
    dist = -torch.cdist(flat, embed[None], p=2)
    ind = dist.argmax(dim=-1)
    onehot = torch.nn.functional.one_hot(ind, Kc).type(x.dtype)
    cs = (onehot * wn).sum(dim=1)
    cluster_size = cluster_size * decay + (1 - decay) * cs[0]
    esum = torch.einsum("hnd,hnc->hcd", flat * wn, onehot)[0]
    sm = (cluster_size + eps) / (cluster_size.sum() + Kc * eps) * cluster_size.sum()
    return ind[0], embed * decay + (1 - decay) * esum / sm[:, None], cluster_size


def test_full_size_iteration_against_the_torch_formulation():
    n, d, Kc = 80000, 27, 8192
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(n, d, device="cuda", generator=g) * 0.5
    embed = torch.randn(Kc, d, device="cuda", generator=g) * 0.5
    w = torch.rand(n, device="cuda", generator=g) ** 2
    cs0 = torch.rand(Kc, device="cuda", generator=g) * 5
    ref_ind, ref_embed, ref_cs = _torch_reference_iteration(x, w, embed, cs0)
    model = vt.VectorQuantize(dim=d, codebook_size=Kc).cuda().train()
    model._codebook.embed.copy_(embed[None])
    model._codebook.cluster_size.copy_(cs0[None])
    _, ind, _ = model(x[None], weight=w.reshape(1, -1, 1))
    ours, refi = ind[0].cpu().numpy(), ref_ind.cpu().numpy()
    assert _ties_only(x.cpu().numpy(), embed.cpu().numpy(), ours, refi)
    assert (ours != refi).mean() < 2e-3
    if (ours != refi).sum() == 0:
        torch.testing.assert_close(model._codebook.cluster_size[0], ref_cs, rtol=1e-4, atol=1e-4)
        torch.testing.assert_close(model._codebook.embed[0], ref_embed, rtol=1e-4, atol=2e-5)
    else:                                                       # a few tie flips move single samples between clusters
        rel = (model._codebook.embed[0] - ref_embed).norm() / ref_embed.norm()
        assert float(rel) < 1e-2


def test_cpu_tensors_are_refused():
    with pytest.raises(RuntimeError):
        vt.vq_assign(torch.zeros(4, 27), torch.zeros(8, 27))


def test_tensor_core_search_equals_the_fp32_kernel_at_full_size():
    """80 000 x 8192 x 27 (vectree/vq.py's chunk): the tensor-core (wgmma) coarse pass + exact rescore of the undecided rows must return the FP32
    kernel's indices -- both kernels break exact ties towards the smaller index; rows whose two best codes differ by less than the fp32
    rounding of the expansion may legitimately differ and are checked in float64"""
    from lightgaussian_b200 import capi
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(80000, 27, device="cuda", generator=g) * 0.5
    e = torch.randn(8192, 27, device="cuda", generator=g) * 0.7
    capi.set_vq_mode(1)
    try:
        ref = vt.vq_assign(x, e).cpu().numpy()
    finally:
        capi.set_vq_mode(0)
    got = vt.vq_assign(x, e).cpu().numpy()
    assert _ties_only(x.cpu().numpy(), e.cpu().numpy(), got, ref)
    assert (got != ref).mean() < 1e-4
    # clustered data (what k-means converges to): many samples sit next to their code, runner-ups are far
    centers = torch.randn(8192, 27, device="cuda", generator=g)
    xc = centers[torch.randint(0, 8192, (80000,), device="cuda", generator=g)] + 0.05 * torch.randn(80000, 27, device="cuda", generator=g)
    capi.set_vq_mode(1)
    try:
        ref = vt.vq_assign(xc, centers).cpu().numpy()
    finally:
        capi.set_vq_mode(0)
    got = vt.vq_assign(xc, centers).cpu().numpy()
    assert _ties_only(xc.cpu().numpy(), centers.cpu().numpy(), got, ref)
    assert (got != ref).mean() < 1e-4
