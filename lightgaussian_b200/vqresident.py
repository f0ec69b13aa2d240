"""A VecTree-compressed model kept resident on the GPU in its compressed form, and rendered from it.

`GaussianModel.load_vq` (scene/gaussian_model.py:420-461) inflates `extreme_saving/` (vectree/vectree.py:107-155) into a dense
[P, 6+D+8] float32 table (vectree/utils.py:5-65) and then into six float32 leaves: 236 B per Gaussian at SH degree 3.  `ResidentVQ`
keeps what the files hold instead: float32 xyz, the fp16 (or float32) attribute rows, one int32 slot per Gaussian, the fp16
codebook and the rows of the Gaussians that were not quantised -- about 70 B per Gaussian with the reference's settings.
`lgr_forward_vq` renders that in place, bit-identically to the leaves (csrc/lgr_raw.cuh, VqSource).

`install(GaussianModel)` makes `load_vq` load a store and defer the five leaves it does not need for rendering; the first read of one
of them (a getter, capture(), save_ply(), training_setup(), a render with gradients) materialises all five exactly as the
reference builds them, and the object is a plain GaussianModel again.
"""
from __future__ import annotations

import math
import os

import numpy as np
import torch
from torch import nn

from . import trace
from .vectree import load_vqgaussian, unpack_indices

_DEFERRED = ("_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity")


def _npz(ex, name, key="arr_0", allow_pickle=False):
    with np.load(os.path.join(ex, name), allow_pickle=allow_pickle) as z:
        return z[key]


def _padded(a, Dp):
    """rows padded with zeros to Dp elements, so that every row starts 16-byte aligned"""
    if a.shape[1] == Dp:
        return np.ascontiguousarray(a)
    out = np.zeros((a.shape[0], Dp), dtype=a.dtype)
    out[:, :a.shape[1]] = a
    return out


class ResidentVQ:
    """The arrays lgr_forward_vq reads (include/lgrast.h, lgr_vq_resident_params), on one CUDA device."""

    def __init__(self, path, max_sh_degree, xyz, attr, slot, codebook, nonvq, D):
        self.path, self.max_sh_degree = path, max_sh_degree
        self.xyz, self.attr, self.slot, self.codebook, self.nonvq = xyz, attr, slot, codebook, nonvq
        self.P, self.D, self.Dp, self.K = xyz.shape[0], D, codebook.shape[1], codebook.shape[0]

    @classmethod
    def load(cls, path, max_sh_degree, device="cuda"):
        """Read `<path>/extreme_saving/*.npz` (the directory GaussianModel.load_vq takes).  Every shape and dtype is checked on the
        host first: a file that disagrees with metadata.npz or with `max_sh_degree` raises ValueError before any GPU work."""
        ex = os.path.join(path, "extreme_saving")
        meta = _npz(ex, "metadata.npz", "metadata", allow_pickle=True).item()
        K, D = int(meta["codebook_size"]), int(meta["codebook_dim"])
        P, dim = int(meta["input_pc_num"]), int(meta["input_pc_dim"])
        if D != 3 * (max_sh_degree + 1) ** 2:
            raise ValueError(f"extreme_saving: codebook_dim {D} does not hold SH degree {max_sh_degree} (needs {3 * (max_sh_degree + 1) ** 2})")
        if dim != 6 + D + 8:
            raise ValueError(f"extreme_saving: input_pc_dim {dim} is not xyz, normals, {D} SH values and 8 attributes")
        bits = int(math.log2(K)) if K > 0 else 0
        if K < 1 or 2 ** bits != K:
            raise ValueError(f"extreme_saving: codebook_size {K} is not a power of two")
        codebook = _npz(ex, "codebook.npz")
        if codebook.dtype != np.float16:
            raise ValueError(f"extreme_saving: the codebook is {codebook.dtype}, the writer stores float16")
        if codebook.shape != (K, D):
            raise ValueError(f"extreme_saving: codebook shape {codebook.shape}, metadata says {(K, D)}")
        mask = _npz(ex, "non_vq_mask.npz")
        if mask.dtype != np.uint8 or mask.ndim != 1 or mask.size * 8 < P:
            raise ValueError(f"extreme_saving: non_vq_mask holds {mask.size * 8} bits for {P} Gaussians")
        n_nonvq = int(np.unpackbits(mask)[:P].sum())
        n_vq = P - n_nonvq
        idx = _npz(ex, "vq_indexs.npz")
        if idx.dtype != np.uint8 or idx.ndim != 1 or idx.size * 8 < n_vq * bits:
            raise ValueError(f"extreme_saving: vq_indexs holds {idx.size * 8} bits, {n_vq} indices of {bits} bits need {n_vq * bits}")
        nonvq = _npz(ex, "non_vq_feats.npz")
        if nonvq.shape != (n_nonvq, D) or nonvq.dtype not in (np.float16, np.float32):
            raise ValueError(f"extreme_saving: non_vq_feats is {nonvq.dtype} {nonvq.shape}, expected float16/float32 {(n_nonvq, D)}")
        attr = _npz(ex, "other_attribute.npz")
        if attr.shape != (P, 8) or attr.dtype not in (np.float16, np.float32):
            raise ValueError(f"extreme_saving: other_attribute is {attr.dtype} {attr.shape}, expected float16/float32 {(P, 8)}")
        xyz = _npz(ex, "xyz.npz")
        if xyz.shape != (P, 3) or xyz.dtype.kind != "f":
            raise ValueError(f"extreme_saving: xyz is {xyz.dtype} {xyz.shape}, expected floating {(P, 3)}")

        dev = torch.device(device)
        if dev.type != "cuda":
            raise ValueError("ResidentVQ lives on a CUDA device: there is no CPU renderer")
        # slot: codebook index for quantised Gaussians, -(row in non_vq_feats) - 1 for the others (their rows are in Gaussian order)
        if P:
            is_nonvq = unpack_indices(torch.from_numpy(mask).to(dev), P, 1).bool()
            vq_idx = (unpack_indices(torch.from_numpy(idx).to(dev), n_vq, bits) if n_vq
                      else torch.empty(0, dtype=torch.int32, device=dev))
            slot = torch.cumsum(is_nonvq, 0, dtype=torch.int32).neg_().masked_scatter_(~is_nonvq, vq_idx)
            del is_nonvq, vq_idx
        else:
            slot = torch.empty(0, dtype=torch.int32, device=dev)
        Dp = (D + 7) // 8 * 8
        return cls(path, max_sh_degree,
                   xyz=torch.from_numpy(np.ascontiguousarray(xyz, dtype=np.float32)).to(dev),
                   attr=torch.from_numpy(np.ascontiguousarray(attr)).to(dev),
                   slot=slot,
                   codebook=torch.from_numpy(_padded(codebook, Dp)).to(dev),
                   nonvq=torch.from_numpy(_padded(nonvq, Dp)).to(dev),
                   D=D)

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in (self.xyz, self.attr, self.slot, self.codebook, self.nonvq))

    def materialize(self) -> dict:
        """The six leaves exactly as GaussianModel.load_vq makes them from the same files: float32 nn.Parameters, requires_grad,
        contiguous, the reference's shapes and bits."""
        dev = self.xyz.device
        # the table goes through the host as in the reference, so the GPU never holds it and the leaves at once
        feats = load_vqgaussian(os.path.join(self.path, "extreme_saving"), device=dev).cpu()
        P, sh_dim = feats.shape[0], 3 * (self.max_sh_degree + 1) ** 2 - 3

        def leaf(t, transpose=False):  # upload, then transpose(1, 2).contiguous() on the device: the reference's strides too
            t = t.contiguous().to(dev)
            return nn.Parameter((t.transpose(1, 2).contiguous() if transpose else t).requires_grad_(True))

        return {"_xyz": leaf(feats[:, 0:3]),
                "_features_dc": leaf(feats[:, 6:9].reshape(P, 3, 1), transpose=True),
                "_features_rest": leaf(feats[:, 9:9 + sh_dim].reshape(P, 3, sh_dim // 3), transpose=True),
                "_opacity": leaf(feats[:, -8:-7]),
                "_scaling": leaf(feats[:, -7:-4]),
                "_rotation": leaf(feats[:, -4:])}


# ---- deferred leaves on a GaussianModel ----
class _DeferredLeaf:
    """Data descriptor of one deferred leaf: reading or assigning it materialises all five and drops the store."""

    def __init__(self, name):
        self.name = name

    def __get__(self, obj, owner=None):
        if obj is None:
            return self
        materialize(obj)
        return getattr(obj, self.name)

    def __set__(self, obj, value):
        materialize(obj)
        setattr(obj, self.name, value)


_subclasses = {}


def _resident_class(base):
    if base not in _subclasses:
        ns = {n: _DeferredLeaf(n) for n in _DEFERRED}
        ns["_lgr_resident_base"] = base
        _subclasses[base] = type(base.__name__, (base,), ns)
    return _subclasses[base]


def defer(obj, store: ResidentVQ):
    """Attach `store` to `obj` and defer its five non-position leaves until something reads or assigns one."""
    base = getattr(type(obj), "_lgr_resident_base", type(obj))
    for n in _DEFERRED:
        obj.__dict__.pop(n, None)
    obj.__dict__["_vq_resident"] = store
    obj.__class__ = _resident_class(base)


def materialize(obj):
    """Replace `obj`'s store by the five leaves the reference's load_vq builds; `obj` is of its original class afterwards."""
    store = obj.__dict__.pop("_vq_resident", None)
    base = getattr(type(obj), "_lgr_resident_base", None)
    if base is not None:
        obj.__class__ = base
    if store is None:
        return
    trace.bump("vq_materialize")
    leaves = store.materialize()
    for n in _DEFERRED:
        setattr(obj, n, leaves[n])


def install(cls):
    """Patch cls.load_vq (scene/gaussian_model.py:420-461) to keep the compressed model resident.  Idempotent."""
    if getattr(cls.load_vq, "_lgr_resident", False):
        return

    def load_vq(self, path):
        store = ResidentVQ.load(path, self.max_sh_degree, "cuda")
        self.active_sh_degree = self.max_sh_degree
        self._xyz = nn.Parameter(store.xyz.requires_grad_(True))
        defer(self, store)

    load_vq._lgr_resident = True
    load_vq._lgr_dense = cls.load_vq   # the class's own load_vq (tests compare against it)
    load_vq.__doc__ = install.__doc__
    cls.load_vq = load_vq
