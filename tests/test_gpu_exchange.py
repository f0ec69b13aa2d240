"""The view-parallel gradient exchange at 1-8 ranks, simulated on ONE GPU.

The exchange kernels take raw device pointers and nothing in them needs the buffers to sit on different GPUs, so N ranks' exchange
buffers are allocated on one device, every rank's pack runs, then every rank's accumulate: exactly the device code of an N-GPU step
(the cross-GPU barrier is only an ordering point), minus NVLink.

  sparse exchange (the default; csrc/lgr_sparse.cuh) through the production marshalling (rasterizer._exchange_tables, _sparse_pack,
  _sparse_accumulate), every view packed in push AND pull mode from the same blend-backward state:
    (a) all ranks' outputs bit-identical, push == pull;
    (b) every slot decoded on the host from the layout (header | bitmap | prefix, 64-word padded | 16-float rows): header, popcounts,
        prefix, flags, pads, push copies, NaN sentinels past the rows;
    (c) xyz / scaling / rotation / opacity == a numpy float32 sum of the decoded rows in ascending view order, bit for bit;
    (d) features_dc / features_rest == lgr_sh_grad_from_views over the decoded dRGB, bit for bit;
    (e) every element within the float64 bound of test_gpu_leafgrad.BOUNDS, summed over the views;
    (f) each rank's dL/dmeans2D against its own view's float64 value; (g) every output row written.
  dense fallback (LGR_EXCHANGE=dense): chunked K7+K8, lgr_peer_allreduce over N buffers, and the composed step."""
import math
import os
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from lightgaussian_b200 import capi
from lightgaussian_b200.model import GaussianParams, TorchCamera
from lightgaussian_b200.rasterizer import (GaussianRasterizationSettings, _exchange_chunks, _exchange_tables, _forward_raw_native, _make_view,
                                           _raw_grads_struct, _raw_struct, _sparse_accumulate, _sparse_pack, backward_raw_native,
                                           sh_grad_from_views)
from lightgaussian_b200.synth import camera_from_pose, look_at, make_cameras, make_scene
from tests.test_gpu_leafgrad import BOUNDS, _activated, _raw_np, _student
from tests.util import LEAVES, assert_every_element, leaf_grads_float64, read_state, view_from_camera

pytestmark = pytest.mark.gpu

NAN_BITS = 0x7FC00000                    # torch.full(float("nan")) on the device
SMALL = {"xyz": (3, 6), "scaling": (6, 9), "rotation": (9, 13), "opacity": (13, 14)}   # columns of a 16-float exchanged row


# ------------------------------------------------------------------------------------------------
# the slot layout, restated from the comment and sparse_layout() in csrc/lgr_sparse.cuh
# ------------------------------------------------------------------------------------------------
def _layout(P):
    w32 = (P + 31) // 32
    w32a = (w32 + 63) // 64 * 64
    bitmap = 64
    prefix = bitmap + w32a
    rows = prefix + w32a
    return SimpleNamespace(w32=w32, bitmap=bitmap, prefix=prefix, rows=rows, total=rows + 16 * P)


def _slot_bytes(cap):
    return (int(capi.load().lgr_sparse_exchange_bytes(cap)) + 255) // 256 * 256


def _decode(words, P):
    """one slot (uint32 numpy array, at least up to the end of its rows) -> dict(campos, count, flags [P], rows [count,16])"""
    L = _layout(P)
    count = int(words[3])
    bitmap = words[L.bitmap:L.bitmap + L.w32]
    prefix = words[L.prefix:L.prefix + L.w32]
    bits = np.unpackbits(bitmap.view(np.uint8), bitorder="little").astype(bool)
    pop = bits.reshape(L.w32, 32).sum(1)
    assert count == int(pop.sum()), "header count != bitmap popcount"
    np.testing.assert_array_equal(prefix.astype(np.int64), np.concatenate([[0], np.cumsum(pop)[:-1]]), "prefix != exclusive popcount scan")
    assert not bits[P:].any(), "bits set past P"
    rows = words[L.rows:L.rows + 16 * count].view(np.float32).reshape(count, 16)
    assert np.all(rows[:, 14:].view(np.uint32) == 0), "pad floats of a row are not 0"
    return dict(campos=words[0:3].copy(), count=count, flags=bits[:P], rows=rows)


# ------------------------------------------------------------------------------------------------
# scenes, views, settings
# ------------------------------------------------------------------------------------------------
def _blind_camera(W, H):
    """looks away from the [-1,1]^3 cloud: every Gaussian behind it"""
    R, t = look_at((0.0, 0.0, 5.0), target=(0.0, 0.0, 10.0))
    return camera_from_pose(R, t, W, H, math.radians(60.0))


def _scene(P, seed, layout, cluster):
    """leaves of make_scene(P); `cluster`: the first min(P, 32) Gaussians (one warp) become large splats at the origin, seen by every
    camera of make_cameras past the cloud's silhouette, so that their lanes hold a row in every view"""
    raw = {k: v.copy() for k, v in make_scene(P, sh_degree=3, seed=seed, scale_mult=2.0)["raw"].items()}
    if cluster:
        n = min(P, 32)
        rng = np.random.default_rng(seed + 1)
        raw["xyz"][:n] = (0.05 * rng.standard_normal((n, 3))).astype(np.float32)
        raw["scaling"][:n] = np.log(0.7 + 0.2 * rng.random((n, 3))).astype(np.float32)
        raw["opacity"][:n] = -2.0
    if layout == "student":
        pc = _student(raw)                                        # M = 9 read through a row stride of 45 floats
    else:
        pc = GaussianParams(raw, 3, "cuda", requires_grad=False)
        if layout == "deg1of3":
            pc.active_sh_degree = 1
    return pc


def _settings(cam, deg, bg, mod):
    tcam = TorchCamera(cam, "cuda")
    return GaussianRasterizationSettings(int(cam.image_height), int(cam.image_width), cam.tanfovx, cam.tanfovy,
                                         torch.tensor(bg, dtype=torch.float32, device="cuda"), mod, tcam.world_view_transform,
                                         tcam.full_proj_transform, deg, tcam.camera_center, False, False, False)


def _dpix(seed, H, W, fewer):
    d = np.random.default_rng(seed).standard_normal((3, H, W)).astype(np.float32)
    if fewer:                     # a step whose views flag fewer Gaussians than the first use of the same buffer did
        d[:, :, W // 3:] = 0.0
    return torch.from_numpy(d).cuda()


# ------------------------------------------------------------------------------------------------
# the simulated ranks
# ------------------------------------------------------------------------------------------------
class _Sim:
    """N ranks' exchange buffers (two alternating buffers per rank, push and pull layouts) on one device, laid out for `cap` Gaussians,
    NaN-filled; per rank a namespace with what _sparse_pack / _sparse_accumulate read."""

    def __init__(self, world, P, cap, nbufs=2):
        self.world, self.P, self.slot = world, P, _slot_bytes(cap)
        n = world * self.slot // 4
        self.bufs, self.ranks, self.used = {}, {}, {}
        ws = torch.empty(int(capi.load().lgr_sparse_workspace_bytes(cap)), dtype=torch.uint8, device="cuda")
        for mode in ("push", "pull"):
            self.bufs[mode] = [[torch.full((n,), float("nan"), device="cuda") for _ in range(world)] for _ in range(nbufs)]
            bases = [[b.data_ptr() for b in per_rank] for per_rank in self.bufs[mode]]
            self.ranks[mode] = []
            for r in range(world):
                pack, ptrs = _exchange_tables(bases, r, self.slot, mode == "push")
                self.ranks[mode].append(SimpleNamespace(pack_tables=pack, ptr_tables=ptrs, rank=r, push=mode == "push", ws=ws))
            self.used[mode] = [False] * nbufs

    def slot_words(self, mode, k, q, v):
        """slot v of rank q's buffer k, as int32 words (a view)"""
        w = self.slot // 4
        return self.bufs[mode][k][q][v * w:(v + 1) * w].view(torch.int32)


def _pack_again(xs, k, rs, leaves, radii, geom, g2d):
    """lgr_backward_raw_sparse_pack_push from the accumulators the previous _sparse_pack's blend backward left (no second blend backward,
    whose float atomics would make the two packs differ)"""
    import ctypes as C
    lib = capi.load()
    xyz, rest = leaves[0], leaves[2]
    P, M = xyz.size(0), 1 + rest.size(1)
    view, keep = _make_view(xyz.device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, rs.image_height,
                            rs.image_width, rs.scale_modifier, rs.sh_degree, False, False)
    st = lib.lgr_backward_raw_sparse_pack_push(C.byref(view), P, M, C.byref(_raw_struct(*leaves)), radii.data_ptr(), geom.data_ptr(),
                                               xs.pack_tables[k], len(xs.pack_tables[k]), xs.rank if xs.push else 0, xs.ws.data_ptr(),
                                               g2d.data_ptr(), capi.current_stream_ptr(xyz.device))
    capi.check(st, "lgr_backward_raw_sparse_pack_push")


def _nan_like(t):
    return torch.full(t.shape, float("nan"), device=t.device)


def _step(sim, k, pc, cams, settings, seed, first_use, fewer=False, oracle_views=(), dense=False, upstream=None):
    """one simulated view-parallel step on buffer k: rank v renders cams[v]; returns the per-rank outputs of both modes, the decoded
    slots, the float64 single-view gradients of the views in oracle_views, and (dense=True) the composed dense-fallback step.  The
    upstream gradient of view v is upstream(v, image) if given, else Gaussian noise."""
    leaves = [p.detach() for p in pc.parameters()]
    P, deg = leaves[0].shape[0], pc.active_sh_degree
    world = sim.world
    g2d = {m: [torch.full((P, 3), float("nan"), device="cuda") for _ in range(world)] for m in ("push", "pull")}
    exact, drgb_dense, flats, g2d_dense = {}, [], [], []
    for v in range(world):
        cam = cams[v]
        rs = settings(cam, deg)
        with torch.no_grad():
            _, _, R, color, radii, geom, binning, img, _ = _forward_raw_native(False, rs, *leaves)
        dpix = upstream(v, color) if upstream else _dpix(seed * 100 + v, cam.image_height, cam.image_width, fewer)
        del color
        _sparse_pack(sim.ranks["push"][v], k, rs, R, dpix, *leaves, radii, geom, binning, img, g2d["push"][v])
        _pack_again(sim.ranks["pull"][v], k, rs, leaves, radii, geom, g2d["pull"][v])
        if v in oracle_views:
            view = view_from_camera(cam, rs.bg.cpu().numpy(), deg, rs.scale_modifier)
            if R == 0:
                exact[v] = None
            else:
                state = read_state(view, P, R, radii.cpu().numpy(), geom, binning, img)
                exact[v] = leaf_grads_float64(view, _raw_np(leaves), state, dpix.cpu().numpy(), act=_activated(leaves, deg))
            exact.setdefault("radii", {})[v] = radii.cpu().numpy()
        if dense:
            g, g2, d_rgb, flat = backward_raw_native(rs, R, dpix, *leaves, radii, geom, binning, img, compact=True)
            drgb_dense.append(d_rgb)
            flats.append(flat)
            g2d_dense.append(g2)
        del geom, binning, img                                 # the blobs of the next view take their place
    # (b) before any rank reads the slots: an index word that did not arrive would send the accumulate kernel's loads anywhere
    dec = _check_slots(sim, k, cams, first_use)
    outs = {}
    for mode in ("push", "pull"):
        outs[mode] = []
        for r in range(world):
            g = [_nan_like(t) for t in leaves]
            _sparse_accumulate(sim.ranks[mode][r], k, deg, world, leaves[0], leaves[2], g)
            outs[mode].append(g)
    torch.cuda.synchronize()
    composed = _compose_dense(leaves, cams, settings, deg, drgb_dense, flats) if dense else None
    return dict(outs=outs, g2d=g2d, exact=exact, composed=composed, g2d_dense=g2d_dense, leaves=leaves, deg=deg, dec=dec)


# ------------------------------------------------------------------------------------------------
# the checks
# ------------------------------------------------------------------------------------------------
def _bits(t):
    return t.contiguous().view(torch.int32)


def _check_replicas(res):
    """(a) every rank's six leaves bit-identical, push == pull, and the two packs wrote the same dL/dmeans2D"""
    ref = res["outs"]["push"][0]
    for mode in ("push", "pull"):
        for r, g in enumerate(res["outs"][mode]):
            for n, a, b in zip(LEAVES, g, ref):
                assert torch.equal(_bits(a), _bits(b)), f"{mode} rank {r} {n} differs from push rank 0"
    for a, b in zip(res["g2d"]["push"], res["g2d"]["pull"]):
        assert torch.equal(_bits(a), _bits(b)), "dL/dmeans2D of the push and pull packs differ"


def _check_slots(sim, k, cams, first_use):
    """(b) decode every view's slot; returns the decoded slots (push layout, from rank 0's buffer)"""
    P, world, L = sim.P, sim.world, _layout(sim.P)
    dec = []
    for v in range(world):
        src = sim.slot_words("push", k, 0, v)
        count = int(src[3].item())
        used = L.rows + 16 * count
        for q in range(world):                                                 # push: the same words in every rank's buffer
            assert torch.equal(sim.slot_words("push", k, q, v)[:used], src[:used]), f"push: slot {v} of rank {q} differs from rank 0"
        own = sim.slot_words("pull", k, v, v)
        assert torch.equal(own[:used], src[:used]), f"pull slot {v} differs from the push slot"
        if first_use:
            for q in range(world):
                assert bool((sim.slot_words("push", k, q, v)[used:] == NAN_BITS).all()), f"push slot {v} of rank {q}: written past row {count}"
                if q != v:
                    assert bool((sim.slot_words("pull", k, q, v) == NAN_BITS).all()), f"pull: rank {v} wrote into rank {q}'s buffer"
            assert bool((own[used:] == NAN_BITS).all()), f"pull slot {v}: written past row {count}"
        d = _decode(src[:used].cpu().numpy().view(np.uint32), P)
        np.testing.assert_array_equal(d["campos"], np.ascontiguousarray(cams[v].camera_center, np.float32).view(np.uint32),
                                      f"header campos of slot {v}")
        dec.append(d)
    return dec


def _check_sums(res, dec, P):
    """(c) the small leaves, (d) the SH leaves, (g) every row written -- from the decoded rows"""
    out = [t.cpu().numpy() for t in res["outs"]["push"][0]]
    o = dict(zip(LEAVES, out))
    for n in LEAVES:
        assert not np.isnan(o[n]).any(), f"{n}: a NaN survived (row not written)"
    acc = np.zeros((P, 16), np.float32)
    drgb = np.zeros((len(dec), P, 3), np.float32)
    any_flag = np.zeros(P, bool)
    for v, d in enumerate(dec):                                # ascending view order, flagged views only, from 0
        idx = np.nonzero(d["flags"])[0]
        acc[idx] = acc[idx] + d["rows"]
        drgb[v, idx] = d["rows"][:, 0:3]
        any_flag |= d["flags"]
    for n, (c0, c1) in SMALL.items():
        np.testing.assert_array_equal(o[n].reshape(P, -1).view(np.uint32), acc[:, c0:c1].view(np.uint32),
                                      f"{n} is not the rank-order float32 sum of the rows")
    leaves = res["leaves"]
    campos = torch.from_numpy(np.stack([d["campos"].view(np.float32) for d in dec])).cuda()
    dc, rest = sh_grad_from_views(leaves[0], campos, torch.from_numpy(drgb).cuda(), res["outs"]["push"][0][1], res["outs"]["push"][0][2],
                                  res["deg"])
    np.testing.assert_array_equal(o["features_dc"].view(np.uint32), dc.cpu().numpy().view(np.uint32), "features_dc != lgr_sh_grad_from_views")
    np.testing.assert_array_equal(o["features_rest"].view(np.uint32), rest.cpu().numpy().view(np.uint32),
                                  "features_rest != lgr_sh_grad_from_views")
    for n in LEAVES:
        assert np.all(o[n][~any_flag] == 0), f"{n}: rows no view flagged are not exact zeros"
    nact = (res["deg"] + 1) ** 2 - 1
    assert np.all(o["features_rest"][:, nact:] == 0), "rest coefficients of inactive degrees are not exact zeros"
    return o, any_flag


def _check_flags_cover(dec, exact):
    """(b) the bitmap is a subset of radii > 0, and every Gaussian with a non-zero float64 single-view gradient is flagged"""
    for v, d in enumerate(dec):
        radii = exact["radii"][v]
        assert not (d["flags"] & (radii <= 0)).any(), f"view {v}: a culled Gaussian is flagged"
        e = exact.get(v)
        if e is None:
            assert d["count"] == 0
            continue
        nz = np.zeros(radii.shape[0], bool)
        for n in LEAVES + ("means2D",):
            nz |= (e[n].reshape(radii.shape[0], -1) != 0).any(1)
        assert not (nz & ~d["flags"]).any(), f"view {v}: {int((nz & ~d['flags']).sum())} Gaussians with a gradient are not flagged"


def _sum_bound_check(ours, exacts, tag):
    """(e) |ours - sum_v e_v| <= sum_v (rho |e_v| + alpha max|e_v|), every element"""
    worst = {}
    for n in LEAVES:
        rho, alpha = BOUNDS[n]
        es = [np.asarray(e[n], np.float64) for e in exacts]
        ex = np.sum(es, axis=0)
        bound = np.sum([rho * np.abs(e) + alpha * np.abs(e).max(initial=0.0) for e in es], axis=0)
        err = np.abs(np.asarray(ours[n], np.float64) - ex)
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(err == 0, 0.0, err / bound)
        w = float(r.max(initial=0.0))
        if w > 1.0:
            i = int(np.argmax(r))
            raise AssertionError(f"{tag} {n}: {int((r > 1).sum())} of {r.size} entries outside the float64 bound; worst at "
                                 f"{np.unravel_index(i, ex.shape)}: ours {np.ravel(ours[n])[i]:.9g} exact {ex.ravel()[i]:.9g} ratio {w:.3g}")
        worst[n] = w
    return worst


def _check_means2d(res, any_flag_by_view, tag):
    """(f) each rank's dL/dmeans2D against its own view's float64 value; unflagged rows exact zeros"""
    for v, g in enumerate(res["g2d"]["push"]):
        a = g.cpu().numpy()
        assert not np.isnan(a).any(), f"{tag} rank {v}: dL/dmeans2D row not written"
        assert np.all(a[~any_flag_by_view[v]] == 0) and np.all(a[:, 2] == 0), f"{tag} rank {v}: unflagged dL/dmeans2D rows not zero"
        e = res["exact"].get(v)
        if e is not None:
            assert_every_element(a, e["means2D"], *BOUNDS["means2D"], f"{tag} rank {v} means2D")


def _zeros_like_exact(P, K):
    return dict(xyz=np.zeros((P, 3)), features_dc=np.zeros((P, 1, 3)), features_rest=np.zeros((P, K, 3)), scaling=np.zeros((P, 3)),
                rotation=np.zeros((P, 4)), opacity=np.zeros((P, 1)), means2D=np.zeros((P, 3)))


# ------------------------------------------------------------------------------------------------
# the dense fallback: chunks of K7+K8, our peer all-reduce over N flat buffers, the SH rebuild
# ------------------------------------------------------------------------------------------------
def _peer_allreduce(bufs, n_floats):
    """lgr_peer_allreduce for ranks 0..N-1 in turn over N buffers on one device (the slices of the ranks are disjoint)"""
    import ctypes as C
    lib = capi.load()
    world = len(bufs)
    table = (C.c_void_p * world)(*[b.data_ptr() for b in bufs])
    for r in range(world):
        capi.check(lib.lgr_peer_allreduce(table, r, world, n_floats, capi.current_stream_ptr(bufs[0].device)), "lgr_peer_allreduce")
    torch.cuda.synchronize()


def _compose_dense(leaves, cams, settings, deg, drgb, flats):
    P = leaves[0].shape[0]
    n = (P * 11 + 1023) // 1024 * 1024                     # _SymmExchange's flat size
    bufs = []
    for f in flats:
        b = torch.zeros(n, device="cuda")
        b[:P * 11] = f
        bufs.append(b)
    _peer_allreduce(bufs, n)
    for b in bufs[1:]:
        assert torch.equal(_bits(b), _bits(bufs[0]))
    flat = bufs[0][:P * 11]
    campos = torch.stack([settings(c, deg).campos for c in cams[:len(flats)]])
    dc, rest = sh_grad_from_views(leaves[0], campos, torch.stack(drgb), torch.empty(leaves[1].shape, device="cuda"),
                                  torch.empty(leaves[2].shape, device="cuda"), deg)
    return dict(rotation=flat[:4 * P].view(P, 4), xyz=flat[4 * P:7 * P].view(P, 3), scaling=flat[7 * P:10 * P].view(P, 3),
                opacity=flat[10 * P:].view(P, 1), features_dc=dc, features_rest=rest)


# ------------------------------------------------------------------------------------------------
# the sparse exchange
# ------------------------------------------------------------------------------------------------
W0, H0 = 96, 64
# id: (world, P, layout, W, H, blind camera, cluster, bg, scale_modifier, dense fallback too)
CASES = {
    "w1-control": (1, 4097, "deg3", W0, H0, False, True, (0.0, 0.0, 0.0), 1.0, False),
    "w2-P31": (2, 31, "deg3", W0, H0, False, True, (0.0, 0.0, 0.0), 1.0, True),
    "w3-P33-deg1of3": (3, 33, "deg1of3", W0, H0, False, True, (0.0, 0.0, 0.0), 1.0, True),
    "w5-P1": (5, 1, "deg3", W0, H0, False, True, (0.0, 0.0, 0.0), 1.0, False),
    "w8-P4097-student": (8, 4097, "student", W0, H0, False, True, (0.0, 0.0, 0.0), 1.0, True),
    "w5-P4097-blind": (5, 4097, "deg3", W0, H0, True, True, (0.0, 0.0, 0.0), 1.0, False),
    "w3-P200003": (3, 200_003, "deg3", 160, 120, False, False, (0.0, 0.0, 0.0), 1.0, True),
    "w8-P33-student-settings": (8, 33, "student", W0, H0, False, True, (0.3, 0.1, 0.6), 0.7, False),
    "w3-P4097-deg1of3-blind-settings": (3, 4097, "deg1of3", W0, H0, True, False, (0.3, 0.1, 0.6), 0.7, True),
    "w2-P200003-student": (2, 200_003, "student", 128, 96, False, True, (0.0, 0.0, 0.0), 1.0, False),
}


@pytest.mark.parametrize("case", list(CASES))
def test_sparse_exchange_simulated_ranks(case):
    """three steps on the two alternating buffers (0, 1, 0; the third flags fewer rows than the first left in buffer 0), buffers laid
    out for 1.25 P, NaN-filled buffers and outputs, checks (a)-(g) at every step, the dense fallback's composed step against the same
    float64 bound"""
    world, P, layout, W, H, blind, cluster, bg, mod, dense = CASES[case]
    pc = _scene(P, seed=P + world, layout=layout, cluster=cluster)
    cams = make_cameras(max(world, 2), W, H)[:world]
    if blind:
        cams[world // 2] = _blind_camera(W, H)
    settings = lambda cam, deg: _settings(cam, deg, bg, mod)  # noqa: E731
    sim = _Sim(world, P, int(P * 1.25))
    K = pc._features_rest.shape[1]
    counts = []
    for s, k in enumerate((0, 1, 0)):
        tag = f"{case} step {s}"
        first = not sim.used["push"][k]
        res = _step(sim, k, pc, cams, settings, seed=s, first_use=first, fewer=(s == 2), oracle_views=range(world), dense=dense and s == 0)
        sim.used["push"][k] = sim.used["pull"][k] = True
        _check_replicas(res)
        dec = res["dec"]
        _check_flags_cover(dec, res["exact"])
        ours, any_flag = _check_sums(res, dec, P)
        counts.append([d["count"] for d in dec])
        exacts = [res["exact"][v] if res["exact"][v] is not None else _zeros_like_exact(P, K) for v in range(world)]
        worst = _sum_bound_check(ours, exacts, tag)
        _check_means2d(res, [d["flags"] for d in dec], tag)
        if cluster and not blind:
            percount = np.sum([d["flags"] for d in dec], axis=0)
            assert percount.max() == world, f"{tag}: no Gaussian holds a row in every view"
        if blind:
            assert dec[world // 2]["count"] == 0
        print(f"\n{tag}: rows per view {counts[-1]}, worst ratio to the bound " + ", ".join(f"{n} {w:.3f}" for n, w in worst.items()))
        if res["composed"] is not None:
            comp = {n: t.cpu().numpy() for n, t in res["composed"].items()}
            wd = _sum_bound_check(comp, exacts, tag + " dense fallback")
            for v, g in enumerate(res["g2d_dense"]):
                if res["exact"][v] is not None:
                    assert_every_element(g.cpu().numpy(), res["exact"][v]["means2D"], *BOUNDS["means2D"], f"{tag} dense rank {v} means2D")
            diff = {n: float(np.abs(comp[n].astype(np.float64) - ours[n]).max(initial=0.0)) for n in LEAVES}
            print(f"{tag}: dense fallback worst ratio " + ", ".join(f"{n} {w:.3f}" for n, w in wd.items()) +
                  "; largest |dense - sparse| " + ", ".join(f"{n} {d:.2e}" for n, d in diff.items()))
    assert sum(counts[2]) <= sum(counts[0])
    if P > 4096:
        assert sum(counts[2]) < sum(counts[0]), "the third step should flag fewer rows than the first use of buffer 0"


def test_sparse_exchange_deterministic_mode_bit_identical():
    """LGR_DETERMINISTIC=1: two whole simulated steps (forward, blend backward, packs, accumulates) give the same bits"""
    world, P = 3, 4097
    pc = _scene(P, seed=5, layout="deg3", cluster=True)
    cams = make_cameras(world, W0, H0)
    settings = lambda cam, deg: _settings(cam, deg, (0.0, 0.0, 0.0), 1.0)  # noqa: E731
    old = os.environ.get("LGR_DETERMINISTIC")
    os.environ["LGR_DETERMINISTIC"] = "1"
    try:
        runs = []
        for rep in range(2):
            sim = _Sim(world, P, P, nbufs=1)
            runs.append(_step(sim, 0, pc, cams, settings, seed=7, first_use=True))
    finally:
        if old is None:
            os.environ.pop("LGR_DETERMINISTIC", None)
        else:
            os.environ["LGR_DETERMINISTIC"] = old
        capi.set_deterministic(False)
    for mode in ("push", "pull"):
        for r in range(world):
            for n, a, b in zip(LEAVES, runs[0]["outs"][mode][r], runs[1]["outs"][mode][r]):
                assert torch.equal(_bits(a), _bits(b)), f"{mode} rank {r} {n}: two deterministic steps differ"
            assert torch.equal(_bits(runs[0]["g2d"][mode][r]), _bits(runs[1]["g2d"][mode][r]))
    _check_replicas(runs[0])


ORACLE_VIEWS = (0, 1)     # the float64 oracle at 3M / 1080p: a few seconds of CPU per view


def test_sparse_exchange_bench_size_world8():
    """3M Gaussians, 1920x1080, views 0-7 of make_cameras(16), bench.py's L1 upstream gradient sign(image - target) / N against its seeded
    targets: checks (a)-(d), (g); the float64 check on view 0's rows and dL/dmeans2D (the bounds are the ones calibrated on this step)"""
    world, P, W, H = 8, 3_000_000, 1920, 1080
    raw = make_scene(P, sh_degree=3, seed=0)["raw"]
    pc = GaussianParams(raw, 3, "cuda", requires_grad=False)
    del raw
    cams = make_cameras(16, W, H)[:world]
    settings = lambda cam, deg: _settings(cam, deg, (0.0, 0.0, 0.0), 1.0)  # noqa: E731
    gen = torch.Generator().manual_seed(1234)
    targets = [torch.rand(3, H, W, generator=gen) for _ in range(world)]

    def l1_upstream(v, image):
        return torch.sign(image - targets[v].cuda()) / float(3 * H * W)
    sim = _Sim(world, P, P, nbufs=1)
    t0 = time.time()
    res = _step(sim, 0, pc, cams, settings, seed=11, first_use=True, oracle_views=ORACLE_VIEWS, upstream=l1_upstream)
    t_step = time.time() - t0
    _check_replicas(res)
    dec = res["dec"]
    _check_flags_cover(dec[:len(ORACLE_VIEWS)], res["exact"])
    ours, _ = _check_sums(res, dec, P)
    del ours
    # the oracle views' own rows against their float64 single-view gradients (the rows are what every rank adds)
    for v in ORACLE_VIEWS:
        e, d = res["exact"][v], dec[v]
        idx = np.nonzero(d["flags"])[0]
        for n, (c0, c1) in SMALL.items():
            a = np.zeros((P, c1 - c0), np.float32)
            a[idx] = d["rows"][:, c0:c1]
            assert_every_element(a, e[n].reshape(P, -1), *BOUNDS[n], f"bench view {v} {n}")
        assert_every_element(res["g2d"]["push"][v].cpu().numpy(), e["means2D"], *BOUNDS["means2D"], f"bench view {v} means2D")
    print(f"\nbench size, 8 simulated ranks: rows per view {[x['count'] for x in dec]}; the step with the float64 oracle of views "
          f"{list(ORACLE_VIEWS)} took {t_step:.1f} s")


# ------------------------------------------------------------------------------------------------
# the dense fallback's pieces
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1000, 4097])
def test_chunked_backward_equals_whole_range(P, monkeypatch):
    """lgr_backward_raw_end_range over _exchange_chunks(P) for 1, 2, 3 and 7 chunks == one whole-range compact call, bit for bit,
    every row written (NaN-filled outputs)"""
    import ctypes as C
    lib = capi.load()
    pc = _scene(P, seed=P, layout="deg3", cluster=True)
    leaves = [p.detach() for p in pc.parameters()]
    cam = make_cameras(3, W0, H0)[1]
    rs = _settings(cam, 3, (0.1, 0.2, 0.3), 1.0)
    with torch.no_grad():
        _, _, R, _, radii, geom, binning, img, _ = _forward_raw_native(False, rs, *leaves)
    dpix = _dpix(P, H0, W0, False)
    view, keep = _make_view(dpix.device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, H0, W0, 1.0, 3, False, False)
    d_rgb = torch.full((P, 3), float("nan"), device="cuda")
    stream = capi.current_stream_ptr(dpix.device)
    capi.check(lib.lgr_backward_raw_begin(C.byref(view), P, int(R), radii.data_ptr(), geom.data_ptr(), binning.data_ptr(), img.data_ptr(),
                                          dpix.data_ptr(), d_rgb.data_ptr(), stream), "lgr_backward_raw_begin")
    params = _raw_struct(*leaves)

    def run(chunks):
        flat = torch.full((P * 11,), float("nan"), device="cuda")
        rgb = torch.full((P, 3), float("nan"), device="cuda")
        g2d = torch.full((P, 3), float("nan"), device="cuda")
        g_rot, g_xyz = flat[:4 * P].view(P, 4), flat[4 * P:7 * P].view(P, 3)
        g_scal, g_op = flat[7 * P:10 * P].view(P, 3), flat[10 * P:].view(P, 1)
        grads = _raw_grads_struct(g_xyz, None, None, g_scal, g_rot, g_op, rgb=rgb)
        for c0, cn in chunks:
            capi.check(lib.lgr_backward_raw_end_range(C.byref(view), P, 16, C.byref(params), radii.data_ptr(), geom.data_ptr(), C.byref(grads),
                                                      g2d.data_ptr(), c0, cn, stream), "lgr_backward_raw_end_range")
        torch.cuda.synchronize()
        return flat, rgb, g2d

    whole = run([(0, P)])
    for t in whole:
        assert not torch.isnan(t).any(), "a row of the whole-range call was not written"
    assert torch.equal(_bits(whole[1]), _bits(d_rgb)), "dL/dRGB of K7+K8 != the blend backward's extraction"
    for n in (1, 2, 3, 7):
        monkeypatch.setenv("LGR_EXCHANGE_CHUNKS", str(n))
        chunks = _exchange_chunks(P)
        assert len(chunks) == min(n, (P + 255) // 256) and sum(c for _, c in chunks) == P
        for a, b in zip(run(chunks), whole):
            assert torch.equal(_bits(a), _bits(b)), f"{n} chunks {chunks} differ from the whole range"


def _flat_size_3m():
    return (3_000_000 * 11 + 1023) // 1024 * 1024


@pytest.mark.parametrize("world", [2, 3, 5, 7, 8])
def test_peer_allreduce_simulated_ranks(world):
    """every buffer == the float32 rank-order sum, all buffers identical, the sentinel after n_floats untouched"""
    sizes = sorted({4, 4 * (world - 1), 4 * world + 4, 1_000_004, _flat_size_3m()})
    g = torch.Generator(device="cuda").manual_seed(world)
    for n in sizes:
        bufs = [torch.randn(n + 4, generator=g, device="cuda") for _ in range(world)]
        for b in bufs:
            b[n:] = float("nan")
        if n <= 1_000_004:
            host = [b[:n].cpu().numpy() for b in bufs]
            want = host[0].copy()
            for h in host[1:]:
                want = want + h                                  # float32, rank order
            want_t = torch.from_numpy(want).cuda()
        else:                                                    # same arithmetic on the device for the 3M-sized buffer
            want_t = bufs[0][:n].clone()
            for b in bufs[1:]:
                want_t = want_t + b[:n]
        _peer_allreduce(bufs, n)
        for r, b in enumerate(bufs):
            assert torch.equal(_bits(b[:n]), _bits(want_t)), f"world {world} n {n}: buffer {r} != the rank-order sum"
            assert bool(torch.isnan(b[n:]).all()), f"world {world} n {n}: buffer {r} written past n_floats"
        del bufs


def test_peer_allreduce_rejects_bad_arguments():
    """a count that is not a multiple of 4, more than 8 ranks, a misaligned buffer: an error and no launch"""
    import ctypes as C
    lib = capi.load()
    stream = capi.current_stream_ptr(torch.device("cuda"))
    bufs = [torch.zeros(1024, device="cuda") for _ in range(9)]
    ptrs = [b.data_ptr() for b in bufs]

    def call(p, world, n):
        n0 = capi.launch_count()
        st = lib.lgr_peer_allreduce((C.c_void_p * len(p))(*p), 0, world, n, stream)
        return st, capi.launch_count() - n0
    assert call(ptrs[:2], 2, 1020) == (0, 1)                     # the same buffers, well-formed: one launch
    for p, world, n in ((ptrs[:2], 2, 1022), (ptrs, 9, 1020), ([ptrs[0], ptrs[1] + 4], 2, 1016)):
        st, launches = call(p, world, n)
        assert st != 0 and launches == 0, (world, n, st, launches)
    torch.cuda.synchronize()
