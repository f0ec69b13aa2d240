"""VecTree vector quantisation of the SH features on the fused kernels (SURVEY.md section 8f, row N4).

Mirrors the pieces of the reference's `vectree/` that carry the GPU work, with the same names, argument meaning and state:

* `VectorQuantize(dim, codebook_size, decay=0.8, commitment_weight=1.0, use_cosine_sim=False, threshold_ema_dead_code=0)` with
  `._codebook.embed [1,K,d]`, `._codebook.cluster_size [1,K]`, `.codebook_size`, `.train()/.eval()` and
  `forward(x[1,n,d], weight=[1,n,1]) -> (quantize, embed_ind, loss)`               (vectree/vq.py:179-306, 308-442)
* `Quantization`: `quantize()` (importance top-k split, 1000 EMA k-means iterations on random 80 000-sample chunks with the
  k_expire replacement, encode, `extreme_saving/*.npz`) and `dequantize()`          (vectree/vectree.py:29-207)
* `load_vqgaussian(path, device)`                                                   (vectree/utils.py:5-65)
* `dec2bin`/`bin2dec`'s role is taken by `pack_indices` / `unpack_indices` (bit-identical byte streams).

One k-means iteration is `lgr_vq_assign` (nearest code + weighted sums, no [n,K] matrices) + `lgr_vq_ema_update`; the
reference's cdist / one_hot / einsum formulation moves ~10 GB per iteration for the same result.  Only the configuration the
reference uses is implemented (one head, Euclidean codebook, no k-means init, threshold_ema_dead_code=0): anything else raises.
There is no CPU path.
"""
from __future__ import annotations

import math
import os

import numpy as np
import torch
from torch import nn

from . import capi


def _f32c(t):
    return t.contiguous() if t.dtype == torch.float32 else t.float().contiguous()


def vq_assign(x, embed, weight=None, want_sums=False):
    """idx[n] (int32) of the nearest code; with want_sums also (cluster_batch[K], embed_sum[K,d]) weighted like vq.py:263-296."""
    lib = capi.load()
    if not (x.is_cuda and embed.is_cuda):
        raise RuntimeError("vq_assign needs CUDA tensors: there is no CPU path")
    x, embed = _f32c(x), _f32c(embed)
    n, d = x.shape
    K = embed.shape[0]
    dev = x.device
    idx = torch.empty(n, dtype=torch.int32, device=dev)
    ws = torch.empty(int(lib.lgr_vq_workspace_bytes(n)), dtype=torch.uint8, device=dev)
    cb = es = None
    if want_sums:
        cb = torch.empty(K, dtype=torch.float32, device=dev)
        es = torch.empty(K, d, dtype=torch.float32, device=dev)
    wsum = None
    if weight is not None:
        weight = _f32c(weight).reshape(-1)
        if weight.shape[0] != n:
            raise RuntimeError("vq_assign: one weight per sample expected")
        wsum = weight.sum()
    capi.set_deterministic(capi.deterministic_requested())   # the rasterizer's rule, at the time of the call
    with torch.cuda.device(dev):
        st = lib.lgr_vq_assign(n, d, K, capi.ptr(x), embed.data_ptr(), capi.ptr(weight), capi.ptr(wsum), capi.ptr(idx), capi.ptr(cb), capi.ptr(es),
                               ws.data_ptr(), capi.current_stream_ptr(dev))
    capi.check(st, "lgr_vq_assign")
    return (idx, cb, es) if want_sums else idx


def vq_gather(idx, embed):
    lib = capi.load()
    embed = _f32c(embed)
    n, d = idx.shape[0], embed.shape[1]
    out = torch.empty(n, d, dtype=torch.float32, device=embed.device)
    with torch.cuda.device(embed.device):
        st = lib.lgr_vq_gather(n, d, capi.ptr(idx), embed.data_ptr(), capi.ptr(out), capi.current_stream_ptr(embed.device))
    capi.check(st, "lgr_vq_gather")
    return out


def pack_indices(idx, bits):
    """uint8 CUDA tensor: `bits` bits per index, MSB first, == np.packbits(dec2bin(idx, bits).reshape(-1)) (vectree.py:120-125)"""
    lib = capi.load()
    idx = idx.to(torch.int32).contiguous()
    n = idx.numel()
    out = torch.empty((n * bits + 7) // 8, dtype=torch.uint8, device=idx.device)
    with torch.cuda.device(idx.device):
        st = lib.lgr_vq_pack_indices(n, bits, capi.ptr(idx), capi.ptr(out), capi.current_stream_ptr(idx.device))
    capi.check(st, "lgr_vq_pack_indices")
    return out


def unpack_indices(packed, n, bits):
    """int32 CUDA tensor [n]: bin2dec(np.unpackbits(packed)[:n*bits].reshape(n, bits)) (vectree/utils.py:33-39)"""
    lib = capi.load()
    packed = packed.contiguous()
    if packed.numel() * 8 < n * bits:
        raise RuntimeError("unpack_indices: the byte stream is shorter than n*bits bits")
    out = torch.empty(n, dtype=torch.int32, device=packed.device)
    with torch.cuda.device(packed.device):
        st = lib.lgr_vq_unpack_indices(n, bits, capi.ptr(packed), capi.ptr(out), capi.current_stream_ptr(packed.device))
    capi.check(st, "lgr_vq_unpack_indices")
    return out


def uniform_init(*shape):
    """vq.py:25-28 (same RNG consumption: identical codebooks for the same torch seed)"""
    t = torch.empty(shape)
    nn.init.kaiming_uniform_(t)
    return t


class EuclideanCodebook(nn.Module):
    """vectree/vq.py:179-306 for num_codebooks=1, kmeans_init=False, learnable_codebook=False, sample_codebook_temp=0."""

    def __init__(self, dim, codebook_size, decay=0.8, eps=1e-5, threshold_ema_dead_code=0):
        super().__init__()
        if threshold_ema_dead_code != 0:
            raise NotImplementedError("EuclideanCodebook: only threshold_ema_dead_code=0 (the reference's setting) is implemented")
        self.decay, self.eps, self.codebook_size, self.num_codebooks = decay, eps, codebook_size, 1
        self.threshold_ema_dead_code = 0
        embed = uniform_init(1, codebook_size, dim)
        self.register_buffer("initted", torch.Tensor([True]))
        self.register_buffer("cluster_size", torch.zeros(1, codebook_size))
        self.register_buffer("embed_avg", embed.clone())
        self.register_buffer("embed", embed)

    @torch.no_grad()
    def forward(self, x, weight=None, verbose=False):
        needs_codebook_dim = x.ndim < 4
        flat = x.float().reshape(-1, x.shape[-1])
        w = None if weight is None else weight.reshape(-1)
        embed = self.embed[0]
        if self.training:
            idx, cluster_batch, embed_sum = vq_assign(flat, embed, w, want_sums=True)
        else:
            idx = vq_assign(flat, embed)
        quantize = vq_gather(idx, embed)                       # the PRE-update codebook, as vq.py:282
        if self.training:
            lib = capi.load()
            scratch = torch.empty(1, dtype=torch.float32, device=flat.device)
            with torch.cuda.device(flat.device):
                st = lib.lgr_vq_ema_update(self.codebook_size, embed.shape[1], float(self.decay), float(self.eps), self.cluster_size.data_ptr(),
                                           self.embed.data_ptr(), cluster_batch.data_ptr(), embed_sum.data_ptr(), scratch.data_ptr(),
                                           capi.current_stream_ptr(flat.device))
            capi.check(st, "lgr_vq_ema_update")
        lead = x.shape[:-1] if not needs_codebook_dim else (1,) + tuple(x.shape[:-1])
        quantize = quantize.reshape(*lead, x.shape[-1])
        embed_ind = idx.long().reshape(*lead)
        if needs_codebook_dim:
            quantize, embed_ind = quantize[0], embed_ind[0]
        return quantize, embed_ind


class VectorQuantize(nn.Module):
    """vectree/vq.py:308-442 in the reference's configuration (one head, no projection, channel_last, Euclidean codebook)."""

    def __init__(self, dim, codebook_size, codebook_dim=None, heads=1, decay=0.8, eps=1e-5, kmeans_init=False, use_cosine_sim=False,
                 threshold_ema_dead_code=0, commitment_weight=1.0, orthogonal_reg_weight=0.0, sample_codebook_temp=0.0, **unsupported):
        super().__init__()
        defaults = {"separate_codebook_per_head": False, "channel_last": True, "accept_image_fmap": False,
                    "orthogonal_reg_active_codes_only": False, "orthogonal_reg_max_codes": None, "sync_codebook": False}
        bad = [k for k, v in unsupported.items() if k != "kmeans_iters" and (k not in defaults or v != defaults[k])]
        if heads != 1 or (codebook_dim not in (None, dim)) or kmeans_init or use_cosine_sim or orthogonal_reg_weight or sample_codebook_temp or bad:
            raise NotImplementedError("VectorQuantize: only the configuration vectree.py uses is implemented "
                                      "(heads=1, Euclidean codebook, no k-means init, no orthogonal loss, temperature 0)")
        self.heads, self.eps, self.commitment_weight, self.codebook_size = 1, eps, commitment_weight, codebook_size
        self._codebook = EuclideanCodebook(dim, codebook_size, decay=decay, eps=eps, threshold_ema_dead_code=threshold_ema_dead_code)

    @property
    def codebook(self):
        return self._codebook.embed[0]

    def forward(self, x, weight=None, verbose=False):
        quantize, embed_ind = self._codebook(x, weight, verbose)
        loss = torch.tensor([0.0], device=x.device)
        if self.training:
            xf = x.float()
            quantize = xf + (quantize - xf)                     # straight-through value (vq.py:402)
            if self.commitment_weight > 0:
                loss = loss + torch.nn.functional.mse_loss(quantize, xf) * self.commitment_weight
        return quantize, embed_ind, loss


def load_vqgaussian(path, device="cuda"):
    """vectree/utils.py:5-65: rebuild the [n, dim] attribute table from extreme_saving/*.npz (indices unpacked on the GPU)."""
    def load_f(name, allow_pickle=False, array_name="arr_0"):
        return np.load(os.path.join(path, name), allow_pickle=allow_pickle)[array_name]

    metadata = load_f("metadata.npz", allow_pickle=True, array_name="metadata").item()
    codebook_size, codebook_dim = metadata["codebook_size"], metadata["codebook_dim"]
    bit_length = int(math.log2(codebook_size))
    n, dim = metadata["input_pc_num"], metadata["input_pc_dim"]
    non_vq_mask = unpack_indices(torch.from_numpy(load_f("non_vq_mask.npz")).to(device), n, 1).bool()
    vq_mask = ~non_vq_mask
    vq_elements = int(vq_mask.sum())
    codebook = torch.from_numpy(load_f("codebook.npz")).float().to(device)
    vq_indexs = unpack_indices(torch.from_numpy(load_f("vq_indexs.npz")).to(device), vq_elements, bit_length)
    full_feats = torch.zeros(n, dim, device=device)
    full_feats[:, 0:3] = torch.from_numpy(load_f("xyz.npz")).float().to(device)
    full_feats[:, -8:] = torch.from_numpy(load_f("other_attribute.npz")).float().to(device)
    full_feats[vq_mask, 6:6 + codebook_dim] = vq_gather(vq_indexs, codebook)
    full_feats[non_vq_mask, 6:6 + codebook_dim] = torch.from_numpy(load_f("non_vq_feats.npz")).float().to(device)
    return full_feats


class Quantization:
    """vectree/vectree.py:29-207 on arrays instead of files for the inputs: `feats` is the [n, 6+sh_dim+8] attribute table of
    read_ply_data (x y z nx ny nz | f_dc f_rest | opacity scale rot), `importance` the imp_score array."""

    def __init__(self, feats, importance=None, sh_degree=2, save_path=None, codebook_size=2 ** 13, iteration_num=1000, vq_ratio=0.6,
                 vq_way="half", device="cuda", VQ_CHUNK=80000, k_expire=10):
        self.sh_dim = 3 + 45 if sh_degree == 3 else 3 + 24
        self.device = torch.device(device)
        self.feats_bak = torch.as_tensor(feats, dtype=torch.float32)
        self.feats = self.feats_bak[:, 6:6 + self.sh_dim].to(self.device).contiguous()
        self.importance = None if importance is None else torch.as_tensor(np.asarray(importance))
        self.model_vq = VectorQuantize(dim=self.sh_dim, codebook_size=codebook_size, decay=0.8, commitment_weight=1.0, use_cosine_sim=False,
                                       threshold_ema_dead_code=0).to(self.device)
        self.save_path, self.codebook_size, self.iteration_num = save_path, codebook_size, int(iteration_num)
        self.vq_ratio, self.vq_way, self.VQ_CHUNK, self.k_expire = vq_ratio, vq_way, VQ_CHUNK, k_expire

    def wage_vq(self, feats):
        return feats.half() if self.vq_way == "half" else feats

    def select(self):
        """vectree.py:166-182: the (1-vq_ratio) most important Gaussians keep their features"""
        imp = torch.ones(self.feats.shape[0], dtype=torch.float64) if self.importance is None else self.importance
        _, large_index = torch.topk(imp, k=int(imp.shape[0] * (1 - self.vq_ratio)), largest=True)
        self.non_vq_mask = torch.zeros_like(imp).bool()
        self.non_vq_mask[large_index] = True
        self.vq_mask = ~self.non_vq_mask
        self.tensor_importance = imp
        return self.non_vq_mask

    @torch.no_grad()
    def train_codebook(self):
        """vectree.py:184-205; the sample draw is the reference's `torch.randint` on the CPU generator"""
        self.model_vq.train()
        feats_needs_vq = self.feats[self.vq_mask.to(self.device)].contiguous()
        imp = self.tensor_importance[self.vq_mask].float().to(self.device)
        k = self.k_expire if self.k_expire <= self.model_vq.codebook_size else 0
        cb = self.model_vq._codebook
        for _ in range(self.iteration_num):
            indexes = torch.randint(low=0, high=feats_needs_vq.shape[0], size=[self.VQ_CHUNK]).to(self.device)
            vq_weight = imp[indexes]
            vq_feature = feats_needs_vq[indexes, :]
            self.model_vq(vq_feature.unsqueeze(0), weight=vq_weight.reshape(1, -1, 1))
            if k:
                _, replace_index = torch.topk(cb.cluster_size, k=k, largest=False)
                _, most_important_index = torch.topk(vq_weight, k=k, largest=True)
                cb.embed[:, replace_index, :] = vq_feature[most_important_index, :]

    @torch.no_grad()
    def calc_vector_quantized_feature(self):
        """vectree.py:86-104, one launch over all rows instead of 8192-row chunks"""
        self.model_vq.eval()
        feat, indices, _ = self.model_vq(self.feats.unsqueeze(0))
        self.model_vq.train()
        return feat[0].half().float(), indices[0]

    @torch.no_grad()
    def fully_vq_reformat(self):
        """vectree.py:107-155: encode and write extreme_saving/*.npz (same file names, dtypes and bit layouts)"""
        all_feat, all_indice = self.calc_vector_quantized_feature()
        if self.save_path is not None:
            ex = os.path.join(self.save_path, "extreme_saving")
            os.makedirs(ex, exist_ok=True)
            metadata = {"input_pc_num": self.feats_bak.shape[0], "input_pc_dim": self.feats_bak.shape[1], "codebook_size": self.codebook_size,
                        "codebook_dim": self.sh_dim}
            np.savez_compressed(os.path.join(ex, "metadata.npz"), metadata=metadata)
            vq_mask_dev = self.vq_mask.to(self.device)
            self.codebook_vq_index = all_indice[vq_mask_dev]
            bits = int(math.log2(self.codebook_size))
            np.savez_compressed(os.path.join(ex, "vq_indexs.npz"), pack_indices(self.codebook_vq_index, bits).cpu().numpy())
            np.savez_compressed(os.path.join(ex, "codebook.npz"), self.model_vq._codebook.embed.cpu().half().numpy().squeeze(0))
            np.savez_compressed(os.path.join(ex, "non_vq_mask.npz"), pack_indices(self.non_vq_mask.to(self.device).to(torch.int32), 1).cpu().numpy())
            np.savez_compressed(os.path.join(ex, "non_vq_feats.npz"), self.wage_vq(self.feats_bak[self.non_vq_mask, 6:6 + self.sh_dim]).numpy())
            np.savez_compressed(os.path.join(ex, "other_attribute.npz"), self.wage_vq(self.feats_bak[:, -8:]).numpy())
            np.savez_compressed(os.path.join(ex, "xyz.npz"), self.feats_bak[:, 0:3].numpy())
        return all_feat, all_indice

    def quantize(self):
        self.select()
        self.train_codebook()
        return self.fully_vq_reformat()

    def dequantize(self):
        return load_vqgaussian(os.path.join(self.save_path, "extreme_saving"), device=self.device)
