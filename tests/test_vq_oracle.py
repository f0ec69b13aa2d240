"""CPU: the VecTree oracle (oracle/vq_oracle.py) against the golden produced by the reference's own vectree modules."""
import os

import numpy as np

from oracle import vq_oracle as vo

G = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pyref_vq.npz")))
G["feats_sh"] = G["full_feats"][:, 6:33]   # the VQ'd SH columns of the full feature rows (stored once)
N, D, K, CHUNK, ITERS, KEXP = (int(v) for v in G["cfg"])


def test_kmeans_iterations_follow_the_reference():
    embed = G["embed_init"][0].astype(np.float64)
    cs = np.zeros(K)
    for it in range(ITERS):
        sel = G[f"it{it}_indexes"]
        x, w = G["feats_sh"][sel], G["imp"][sel]
        idx, gap = vo.assign(x, embed)
        ref_idx = G[f"it{it}_ind"]
        bad = idx != ref_idx
        assert np.all(gap[bad] < 1e-4), "assignments may differ from the reference's only at numerical ties"
        if it == 0:
            np.testing.assert_allclose(G["it0_quantize"], embed[ref_idx], rtol=0, atol=1e-6)
            assert abs(vo.commitment_loss(x, embed[ref_idx]) - float(G["it0_loss"][0])) < 1e-5 * float(G["it0_loss"][0])
        _, embed_new, cs = vo.ema_step(x, w, embed, cs, idx=ref_idx)
        np.testing.assert_allclose(cs, G[f"it{it}_cluster_size"][0], rtol=2e-5, atol=1e-4)
        np.testing.assert_allclose(embed_new, G[f"it{it}_embed_after_ema"][0], rtol=1e-4, atol=2e-5)
        cs_ref = G[f"it{it}_cluster_size"][0]
        rep, least, top = vo.replace_least_used(G[f"it{it}_embed_after_ema"][0], cs_ref, x, w, KEXP)
        ref_rep = G[f"it{it}_embed_after_replace"][0]
        changed = np.where(np.any(ref_rep != G[f"it{it}_embed_after_ema"][0], axis=1))[0]
        assert len(changed) == KEXP and np.all(cs_ref[changed] <= np.sort(cs_ref)[KEXP - 1])     # topk may break ties among unused codes differently
        np.testing.assert_array_equal(np.sort(ref_rep[changed], axis=0), np.sort(x[top], axis=0))  # ...but they receive the k most important samples
        embed = ref_rep.astype(np.float64)                             # continue from the reference's state


def test_codec_is_bit_exact():
    idx = G["codec_idx"]
    np.testing.assert_array_equal(vo.pack_indices(idx, 13), G["codec_packed"])
    np.testing.assert_array_equal(vo.unpack_indices(G["codec_packed"], len(idx), 13), G["codec_roundtrip"])
    np.testing.assert_array_equal(G["codec_roundtrip"], idx)


def test_on_disk_format_and_dequantize():
    vq_mask = ~G["non_vq_mask"]
    bits = int(np.log2(K))
    np.testing.assert_array_equal(vo.pack_indices(G["all_indice"][vq_mask], bits), G["file_vq_indexs"])
    np.testing.assert_array_equal(np.packbits(G["non_vq_mask"]), G["file_non_vq_mask"])
    files = {k[5:]: G[k] for k in G if k.startswith("file_") and k != "file_metadata"}
    np.testing.assert_array_equal(vo.dequantize(files, G["file_metadata"]), G["dequantized"])
    # the encode the files came from: nearest code of the (float32) final codebook, features rounded through fp16
    idx, gap = vo.assign(G["feats_sh"], G[f"it{ITERS - 1}_embed_after_replace"][0])
    bad = idx != G["all_indice"]
    assert np.all(gap[bad] < 1e-4)
    np.testing.assert_array_equal(G["all_feat"], G[f"it{ITERS - 1}_embed_after_replace"][0][G["all_indice"]].astype(np.float16).astype(np.float32))
