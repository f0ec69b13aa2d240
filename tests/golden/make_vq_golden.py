"""Generates tests/golden/pyref_vq.npz by IMPORTING the reference's own VecTree modules on CPU (vectree/vq.py, vectree/utils.py,
vectree/vectree.py): per-iteration states of the importance-weighted EMA k-means (VectorQuantize.forward with weight, then the
k_expire replacement of vectree.py:203-205), the final encode, and the on-disk codec (extreme_saving/*.npz written by
Quantization.fully_vq_reformat, read back by load_vqgaussian).
Needs the reference checkout:  python tests/golden/make_vq_golden.py"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "dropin"))          # plyfile shim
sys.path.insert(0, "/root/reference/vectree")            # vq, utils, vectree as the script sees them
import vq as ref_vq                                       # noqa: E402
import utils as ref_utils                                 # noqa: E402
import vectree as ref_vectree                             # noqa: E402

ref_vectree.device = torch.device("cpu")
torch.manual_seed(0)
rng = np.random.default_rng(0)
N, D, K, CHUNK, ITERS, KEXP = 3000, 27, 64, 1024, 6, 4
centers = rng.standard_normal((40, D)).astype(np.float32) * 2.0                       # well separated clusters: stable assignments
feats_sh = (centers[rng.integers(0, 40, N)] + 0.15 * rng.standard_normal((N, D))).astype(np.float32)
imp = (rng.random(N) ** 3 * 1000).astype(np.float32)
out = {"feats_sh": feats_sh, "imp": imp, "cfg": np.array([N, D, K, CHUNK, ITERS, KEXP])}

model = ref_vq.VectorQuantize(dim=D, codebook_size=K, decay=0.8, commitment_weight=1.0, use_cosine_sim=False, threshold_ema_dead_code=0)
out["embed_init"] = model._codebook.embed.numpy().copy()
feats_t, imp_t = torch.from_numpy(feats_sh), torch.from_numpy(imp)
model.train()
with torch.no_grad():
    for it in range(ITERS):
        indexes = torch.randint(low=0, high=N, size=[CHUNK])
        w, x = imp_t[indexes], feats_t[indexes, :]
        quantize, ind, loss = model(x.unsqueeze(0), weight=w.reshape(1, -1, 1))
        out[f"it{it}_indexes"] = indexes.numpy().copy()
        out[f"it{it}_ind"] = ind[0].numpy().copy()
        if it == 0:
            out["it0_quantize"] = quantize[0].numpy().copy()
        out[f"it{it}_loss"] = loss.numpy().copy()
        out[f"it{it}_embed_after_ema"] = model._codebook.embed.numpy().copy()
        out[f"it{it}_cluster_size"] = model._codebook.cluster_size.numpy().copy()
        replace_val, replace_index = torch.topk(model._codebook.cluster_size, k=KEXP, largest=False)
        _, most_important_index = torch.topk(w, k=KEXP, largest=True)
        model._codebook.embed[:, replace_index, :] = x[most_important_index, :]
        out[f"it{it}_embed_after_replace"] = model._codebook.embed.numpy().copy()

# ---- encode + on-disk format through the reference's own Quantization methods (constructed without its PLY-reading __init__) ----
q = object.__new__(ref_vectree.Quantization)
full = np.zeros((N, 6 + D + 8), np.float32)
full[:, 0:3] = rng.standard_normal((N, 3))
full[:, 6:6 + D] = feats_sh
full[:, -8:] = rng.standard_normal((N, 8))
q.feats_bak = torch.from_numpy(full)
q.feats = q.feats_bak[:, 6:6 + D]
q.sh_dim, q.model_vq, q.codebook_size, q.vq_way = D, model, K, "half"
tensor_importance = imp_t
large_val, large_index = torch.topk(tensor_importance, k=int(N * (1 - 0.6)), largest=True)
q.all_one_mask = torch.ones_like(tensor_importance).bool()
q.non_vq_mask = torch.zeros_like(tensor_importance).bool()
q.non_vq_mask[large_index] = True
def _zip_with_python(cmd):            # the `zip` binary is absent in this image: do what `zip -r X.zip X` does, for the size print-out only
    import shutil
    target = cmd.split()[2]
    shutil.make_archive(target[:-4], "zip", os.path.dirname(target), "extreme_saving")
    return 0


with tempfile.TemporaryDirectory() as tmp:
    q.save_path = tmp
    real_system, os.system = os.system, _zip_with_python
    try:
        all_feat, all_indice = q.fully_vq_reformat()
    finally:
        os.system = real_system
    ex = os.path.join(tmp, "extreme_saving")
    for name in ["vq_indexs", "codebook", "non_vq_mask", "non_vq_feats", "other_attribute", "xyz"]:
        out[f"file_{name}"] = np.load(os.path.join(ex, name + ".npz"))["arr_0"]
    out["file_metadata"] = np.array([N, full.shape[1], K, D])
    out["dequantized"] = ref_utils.load_vqgaussian(ex, device="cpu").numpy()
out["full_feats"] = full
out["all_feat"] = all_feat.numpy()
out["all_indice"] = all_indice.numpy()
out["non_vq_mask"] = q.non_vq_mask.numpy()
# codec alone, odd sizes
idx = rng.integers(0, 2 ** 13, 1001)
out["codec_idx"] = idx
out["codec_packed"] = np.packbits(ref_utils.dec2bin(torch.from_numpy(idx), 13).bool().numpy().reshape(-1))
out["codec_roundtrip"] = ref_utils.bin2dec(torch.from_numpy(np.unpackbits(out["codec_packed"])[:1001 * 13].reshape(1001, 13)).float(), 13).long().numpy()
assert np.array_equal(out["full_feats"][:, 6:6 + D], out.pop("feats_sh"))   # the readers take it from full_feats (keeps the file < 1 MB)
np.savez_compressed(os.path.join(HERE, "pyref_vq.npz"), **out)
print("ok", {k: v.shape for k, v in out.items() if k.startswith(("file_", "all_", "deq"))})
