"""View-parallel densification statistics (densify.add_densification_stats with enable_gradient_exchange(world, densification=True)),
1-8 ranks simulated on ONE GPU as tests/test_gpu_exchange.py does: every rank's pack, then every rank's statistics call, on exchange
buffers that all sit on one device.

  wire format   word 14 of every row = the numpy float32 norm of that view's dL/dmeans2D, word 15 zero, the visibility bitmap after
                the rows = packed radii > 0, push copies identical, header flag / serial / P
  sums          every rank's accum / denom bit-identical, == a numpy float32 sequential emulation over the views in rank order, ==
                lgr_densify_stats view after view, == the all-gather path (encode -> stack -> add views)
  serial        == one process that runs backward_raw_native per view and add_densification_stats after each (deterministic mode)
  validation    a wrong filter, another view's gradient, a stale buffer, a pack without statistics: densify_and_prune raises
  replicas      three simulated replicas through two densify events stay bit-identical
"""
import ctypes as C
import os
import socket
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from lightgaussian_b200 import capi, densify, rasterizer
from lightgaussian_b200.model import GaussianParams
from lightgaussian_b200.optim import _GROUP_ATTR
from lightgaussian_b200.rasterizer import (_exchange_tables, _forward_raw_native, _make_view, _raw_struct, _sparse_accumulate, _sparse_pack,
                                           backward_raw_native)
from lightgaussian_b200.synth import make_cameras, make_scene
from tests.test_gpu_exchange import _blind_camera, _dpix, _scene, _settings

pytestmark = pytest.mark.gpu

MAGIC = 0x53544154
W0, H0 = 96, 64


# ------------------------------------------------------------------------------------------------
# the stats slot, restated from lgr_sparse.cuh
# ------------------------------------------------------------------------------------------------
def _layout(P):
    w32 = (P + 31) // 32
    w32a = (w32 + 63) // 64 * 64
    rows = 64 + 2 * w32a
    return SimpleNamespace(w32=w32, bitmap=64, prefix=64 + w32a, rows=rows, vis=rows + 16 * P, total=rows + 16 * P + w32a)


class _StatsSim:
    """N ranks' stats-carrying exchange buffers on one device (push and pull layouts), NaN-filled"""

    def __init__(self, world, P, cap, nbufs=2, modes=("push", "pull")):
        lib = capi.load()
        self.world, self.P = world, P
        self.slot = (int(lib.lgr_sparse_exchange_bytes_stats(cap)) + 255) // 256 * 256
        assert self.slot >= _layout(cap).total * 4
        n = world * self.slot // 4
        ws = torch.empty(int(lib.lgr_sparse_workspace_bytes(cap)), dtype=torch.uint8, device="cuda")
        self.bufs, self.ranks = {}, {}
        for mode in modes:
            self.bufs[mode] = [[torch.full((n,), float("nan"), device="cuda") for _ in range(world)] for _ in range(nbufs)]
            bases = [[b.data_ptr() for b in per_rank] for per_rank in self.bufs[mode]]
            self.ranks[mode] = []
            for r in range(world):
                pack, ptrs = _exchange_tables(bases, r, self.slot, mode == "push")
                self.ranks[mode].append(SimpleNamespace(pack_tables=pack, ptr_tables=ptrs, rank=r, push=mode == "push", ws=ws, stats=True))

    def slot_words(self, mode, k, q, v):
        w = self.slot // 4
        return self.bufs[mode][k][q][v * w:(v + 1) * w].view(torch.int32)


def _pack_again(xs, k, rs, leaves, radii, geom, g2d, serial):
    """the stats pack from the accumulators the previous pack's blend backward left (a second blend backward could differ)"""
    lib = capi.load()
    xyz, rest = leaves[0], leaves[2]
    P, M = xyz.size(0), 1 + rest.size(1)
    view, keep = _make_view(xyz.device, rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos, rs.tanfovx, rs.tanfovy, rs.image_height,
                            rs.image_width, rs.scale_modifier, rs.sh_degree, False, False)
    stats = capi.LgrSparseStats(serial)
    capi.check(lib.lgr_backward_raw_sparse_pack_push_ex(C.byref(view), P, M, C.byref(_raw_struct(*leaves)), radii.data_ptr(), geom.data_ptr(),
                                                        xs.pack_tables[k], len(xs.pack_tables[k]), xs.rank if xs.push else 0, xs.ws.data_ptr(),
                                                        g2d.data_ptr(), C.byref(stats), capi.current_stream_ptr(xyz.device)),
               "lgr_backward_raw_sparse_pack_push_ex")


def _pack_views(sim, k, serial, leaves, deg, cams, settings, dpix_of, modes=("push", "pull"), stats=True):
    """every simulated rank v renders cams[v] and packs it into buffer k; returns per mode the g2d of every rank and the radii"""
    P, world = leaves[0].shape[0], sim.world
    g2d = {m: [torch.full((P, 3), float("nan"), device="cuda") for _ in range(world)] for m in modes}
    radii_all = []
    for v in range(world):
        rs = settings(cams[v], deg)
        with torch.no_grad():
            _, _, R, color, radii, geom, binning, img, _ = _forward_raw_native(False, rs, *leaves)
        dpix = dpix_of(v, color)
        first = modes[0]
        _sparse_pack(sim.ranks[first][v], k, rs, R, dpix, *leaves, radii, geom, binning, img, g2d[first][v], serial=serial if stats else None)
        for m in modes[1:]:
            _pack_again(sim.ranks[m][v], k, rs, leaves, radii, geom, g2d[m][v], serial)
        radii_all.append(radii)
        del geom, binning, img
    return g2d, radii_all


def _np_norm(g):
    a, b = g[:, 0].astype(np.float32), g[:, 1].astype(np.float32)
    return np.sqrt((a * a).astype(np.float32) + (b * b).astype(np.float32)).astype(np.float32)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _seeded_stats(P, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    accum = (torch.rand((P, 1), generator=g, device="cuda") * 3.0).contiguous()
    denom = torch.randint(0, 50, (P, 1), generator=g, device="cuda").float().contiguous()
    return accum, denom


def _run_exchanged(xs, k, rank, serial, world, g2d, filt, accum, denom):
    a, d = accum.clone(), denom.clone()
    densify.stats_exchanged(xs, k, rank, serial, world, g2d, filt, a, d)
    return a, d


def _emulate(accum, denom, g2ds, filts):
    """numpy float32, views in rank order: accum += |g[:2]| and denom += 1 on each view's filter"""
    acc, den = accum.cpu().numpy()[:, 0].copy(), denom.cpu().numpy()[:, 0].copy()
    for g, f in zip(g2ds, filts):
        n = _np_norm(g.cpu().numpy())
        f = f.cpu().numpy()
        acc[f] = (acc[f] + n[f]).astype(np.float32)
        den[f] = (den[f] + np.float32(1.0)).astype(np.float32)
    return acc, den


def _serial_native(accum, denom, g2ds, filts):
    a, d = accum.clone(), denom.clone()
    holder = SimpleNamespace(xyz_gradient_accum=a, denom=d)
    for g, f in zip(g2ds, filts):
        densify.add_densification_stats(holder, SimpleNamespace(grad=g), f)
    return a, d


def _generic(accum, denom, g2ds, filts):
    views = torch.stack([densify.stats_encode(g, f) for g, f in zip(g2ds, filts)])
    a, d = accum.clone(), denom.clone()
    densify.stats_add_views(views, a, d)
    return a, d


# ------------------------------------------------------------------------------------------------
# 1 + 2: wire format and sums
# ------------------------------------------------------------------------------------------------
GRID = [(w, P) for w in (1, 2, 3, 5, 8) for P in (1, 31, 33, 4097, 100_000)]


@pytest.mark.parametrize("world,P", GRID, ids=[f"w{w}-P{P}" for w, P in GRID])
def test_stats_wire_format_and_sums(world, P):
    pc = _scene(P, seed=P + 7 * world, layout="deg3", cluster=True)
    leaves = [p.detach() for p in pc.parameters()]
    cams = make_cameras(max(world, 2), W0, H0)[:world]
    cams[world // 2] = _blind_camera(W0, H0)
    settings = lambda cam, deg: _settings(cam, deg, (0.0, 0.0, 0.0), 1.0)  # noqa: E731
    sim = _StatsSim(world, P, int(P * 1.25) + 1)
    serial, k = 1234567 + world, 1
    L = _layout(P)
    g2d, radii = _pack_views(sim, k, serial, leaves, 3, cams, settings, lambda v, img: _dpix(P * 10 + v, H0, W0, False))
    torch.cuda.synchronize()
    filts = [(r > 0).contiguous() for r in radii]
    assert not filts[world // 2].any(), "the blind view sees something"
    # ---- wire format
    for v in range(world):
        src = sim.slot_words("push", k, 0, v)
        count = int(src[3].item())
        used = L.rows + 16 * count
        for q in range(world):
            w = sim.slot_words("push", k, q, v)
            assert torch.equal(w[:used], src[:used]), f"push copy of slot {v} in rank {q}'s buffer differs"
            assert torch.equal(w[L.vis:L.vis + L.w32], src[L.vis:L.vis + L.w32]), f"push copy of vis {v} in rank {q} differs"
        own = sim.slot_words("pull", k, v, v)
        assert torch.equal(own[:used], src[:used]) and torch.equal(own[L.vis:L.vis + L.w32], src[L.vis:L.vis + L.w32]), "pull != push"
        words = src.cpu().numpy().view(np.uint32)
        assert words[4] == MAGIC and words[5] == serial and words[6] == P, f"slot {v} header {words[:8]}"
        bitmap = np.unpackbits(words[L.bitmap:L.bitmap + L.w32].view(np.uint8), bitorder="little").astype(bool)
        vis = np.unpackbits(words[L.vis:L.vis + L.w32].view(np.uint8), bitorder="little").astype(bool)
        want_vis = radii[v].cpu().numpy() > 0
        assert not vis[P:].any(), "vis bits past P"
        np.testing.assert_array_equal(vis[:P], want_vis, f"slot {v}: vis != radii > 0")
        assert not (bitmap[:P] & ~vis[:P]).any()
        rows = words[L.rows:L.rows + 16 * count].reshape(count, 16)
        idx = np.nonzero(bitmap[:P])[0]
        g = g2d["push"][v].cpu().numpy()
        np.testing.assert_array_equal(rows[:, 14], _np_norm(g[idx]).view(np.uint32), f"slot {v}: word 14 != |dL/dmeans2D|")
        assert np.all(rows[:, 15] == 0), f"slot {v}: word 15 not zero"
        assert torch.equal(_bits(g2d["push"][v]), _bits(g2d["pull"][v]))
    # ---- sums
    accum, denom = _seeded_stats(P, seed=world * 31 + P)
    outs = []
    for mode in ("push", "pull"):
        for r in range(world):
            outs.append(_run_exchanged(sim.ranks[mode][r], k, r, serial, world, g2d[mode][r], filts[r], accum, denom))
    err = densify.error_word(torch.device("cuda"))
    assert int(err.item()) == 0, f"error word {int(err.item())}"
    for a, d in outs[1:]:
        assert torch.equal(_bits(a), _bits(outs[0][0])) and torch.equal(_bits(d), _bits(outs[0][1])), "ranks differ"
    ea, ed = _emulate(accum, denom, g2d["push"], filts)
    np.testing.assert_array_equal(outs[0][0].cpu().numpy()[:, 0].view(np.uint32), ea.view(np.uint32), "accum != numpy emulation")
    np.testing.assert_array_equal(outs[0][1].cpu().numpy()[:, 0].view(np.uint32), ed.view(np.uint32), "denom != numpy emulation")
    sa, sd = _serial_native(accum, denom, g2d["push"], filts)
    assert torch.equal(_bits(sa), _bits(outs[0][0])) and torch.equal(_bits(sd), _bits(outs[0][1])), "!= lgr_densify_stats view by view"
    ga, gd = _generic(accum, denom, g2d["push"], filts)
    assert torch.equal(_bits(ga), _bits(outs[0][0])) and torch.equal(_bits(gd), _bits(outs[0][1])), "all-gather path != fast path"


def test_stats_off_slot_unchanged():
    """the stats-off pack keeps its slot size and leaves every row's word 14 zero"""
    lib = capi.load()
    for P in (1, 33, 4097):
        L = _layout(P)
        assert int(lib.lgr_sparse_exchange_bytes(P)) == L.vis * 4
        assert int(lib.lgr_sparse_exchange_bytes_stats(P)) == L.total * 4


# ------------------------------------------------------------------------------------------------
# 3: serial equivalence in deterministic mode
# ------------------------------------------------------------------------------------------------
@pytest.fixture
def deterministic(monkeypatch):
    monkeypatch.setenv("LGR_DETERMINISTIC", "1")
    yield
    capi.set_deterministic(False)


def test_stats_equal_one_process_loop(deterministic):
    world, P = 3, 4097
    pc = _scene(P, seed=11, layout="deg3", cluster=True)
    leaves = [p.detach() for p in pc.parameters()]
    cams = make_cameras(world, W0, H0)
    settings = lambda cam, deg: _settings(cam, deg, (0.0, 0.0, 0.0), 1.0)  # noqa: E731
    sim = _StatsSim(world, P, P, nbufs=1, modes=("push",))
    g2d, radii = _pack_views(sim, 0, 5, leaves, 3, cams, settings, lambda v, img: _dpix(900 + v, H0, W0, False), modes=("push",))
    accum, denom = _seeded_stats(P, seed=3)
    fast = [_run_exchanged(sim.ranks["push"][r], 0, r, 5, world, g2d["push"][r], (radii[r] > 0).contiguous(), accum, denom)
            for r in range(world)]
    # one process: render view after view, the dense backward, the native statistics after each
    a, d = accum.clone(), denom.clone()
    holder = SimpleNamespace(xyz_gradient_accum=a, denom=d)
    for v in range(world):
        rs = settings(cams[v], 3)
        with torch.no_grad():
            _, _, R, color, rad, geom, binning, img, _ = _forward_raw_native(False, rs, *leaves)
        _, g2, _, _ = backward_raw_native(rs, R, _dpix(900 + v, H0, W0, False), *leaves, rad, geom, binning, img)
        assert torch.equal(rad, radii[v])
        assert torch.equal(_bits(g2), _bits(g2d["push"][v])), f"view {v}: the pack's dL/dmeans2D differs from the dense kernel's"
        densify.add_densification_stats(holder, SimpleNamespace(grad=g2), (rad > 0).contiguous())
    assert int(densify.error_word(torch.device("cuda")).item()) == 0
    for fa, fd in fast:
        assert torch.equal(_bits(fa), _bits(a)) and torch.equal(_bits(fd), _bits(d)), "exchanged statistics != the one-process loop"


# ------------------------------------------------------------------------------------------------
# a GaussianModel stand-in: the attributes densify_and_prune reads
# ------------------------------------------------------------------------------------------------
class _Model(GaussianParams):
    def __init__(self, raw, lr=1e-3):
        super().__init__(raw, 3, "cuda", requires_grad=True)
        for n in ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity"):
            setattr(self, n, torch.nn.Parameter(getattr(self, n).detach().clone()))
        groups = [{"params": [getattr(self, attr)], "lr": lr, "name": name} for name, attr in _GROUP_ATTR.items()]
        self.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15)
        self.percent_dense = 0.01
        P = self._xyz.shape[0]
        self.xyz_gradient_accum = torch.zeros((P, 1), device="cuda")
        self.denom = torch.zeros((P, 1), device="cuda")
        self.max_radii2D = torch.zeros((P,), device="cuda")

    def state(self):
        st = [p.detach().clone() for p in self.parameters()]
        for p in self.parameters():
            s = self.optimizer.state.get(p, {})
            st += [s[k].clone() for k in ("exp_avg", "exp_avg_sq") if k in s]
        return st + [self.xyz_gradient_accum.clone(), self.denom.clone(), self.max_radii2D.clone()]


def _same(a, b):
    return len(a) == len(b) and all(x.shape == y.shape and torch.equal(_bits(x), _bits(y)) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------
# 4 + 5: validation, no host synchronisation
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fault", ["filter", "other_view_grad", "stale_buffer", "pack_without_stats"])
def test_inconsistent_stats_call_makes_densify_raise(fault):
    world, P = 2, 4097
    raw = make_scene(P, sh_degree=3, seed=21, scale_mult=2.0)["raw"]
    model = _Model(raw)
    leaves = [p.detach() for p in model.parameters()]
    cams = make_cameras(world, W0, H0)
    settings = lambda cam, deg: _settings(cam, deg, (0.0, 0.0, 0.0), 1.0)  # noqa: E731
    sim = _StatsSim(world, P, P, nbufs=2, modes=("push",))
    dp = lambda v, img: _dpix(40 + v, H0, W0, False)  # noqa: E731
    g2d, radii = _pack_views(sim, 0, 1, leaves, 3, cams, settings, dp, modes=("push",), stats=fault != "pack_without_stats")
    k, serial = 0, 1
    if fault == "stale_buffer":        # the next step went to buffer 1; the call reads buffer 0 with the current serial
        g2d, radii = _pack_views(sim, 1, 2, leaves, 3, cams, settings, dp, modes=("push",))
        k, serial = 0, 2
    filt = (radii[0] > 0).contiguous()
    grad = g2d["push"][0]
    if fault == "filter":
        filt = filt.clone()
        i = int(torch.nonzero(filt)[0].item())
        filt[i] = False
    if fault == "other_view_grad":
        grad = g2d["push"][1]
    densify.error_word(torch.device("cuda")).zero_()
    before = model.state()
    densify.stats_exchanged(sim.ranks["push"][0], k, 0, serial, world, grad, filt, model.xyz_gradient_accum, model.denom)
    P0 = model._xyz.shape[0]
    with pytest.raises(RuntimeError, match="inconsistent across ranks"):
        densify.densify_and_prune(model, 1e-9, 0.005, 1.0, None)
    after = model.state()
    assert model._xyz.shape[0] == P0
    assert _same(before[:-3], after[:-3]), "densify_and_prune changed the model before raising"
    # reported once: the next event runs
    densify.densify_and_prune(model, 1e30, 0.0, 1.0, None)


def test_fast_path_dispatch_without_host_sync():
    """add_densification_stats with the exchange on and a record of this step: the exchanged kernel, no host synchronisation"""
    world, P = 2, 4097
    pc = _scene(P, seed=2, layout="deg3", cluster=True)
    leaves = [p.detach() for p in pc.parameters()]
    cams = make_cameras(world, W0, H0)
    settings = lambda cam, deg: _settings(cam, deg, (0.0, 0.0, 0.0), 1.0)  # noqa: E731
    sim = _StatsSim(world, P, P, nbufs=1, modes=("push",))
    g2d, radii = _pack_views(sim, 0, 9, leaves, 3, cams, settings, lambda v, img: _dpix(70 + v, H0, W0, False), modes=("push",))
    accum, denom = _seeded_stats(P, seed=8)
    want = _emulate(accum, denom, g2d["push"], [(r > 0) for r in radii])
    holder = SimpleNamespace(xyz_gradient_accum=accum.clone(), denom=denom.clone())
    vs = SimpleNamespace(grad=g2d["push"][1])
    filt = (radii[1] > 0).contiguous()
    densify.error_word(torch.device("cuda")).zero_()
    rasterizer.enable_gradient_exchange(world, densification=True)
    try:
        rasterizer._exchange["stats_record"] = dict(xs=sim.ranks["push"][1], k=0, serial=9, P=P, device=accum.device)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            densify.add_densification_stats(holder, vs, filt)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert rasterizer._exchange["stats_record"] is None, "the record was not consumed"
    finally:
        rasterizer.enable_gradient_exchange(1)
    assert int(densify.error_word(torch.device("cuda")).item()) == 0
    np.testing.assert_array_equal(holder.xyz_gradient_accum.cpu().numpy()[:, 0].view(np.uint32), want[0].view(np.uint32))
    np.testing.assert_array_equal(holder.denom.cpu().numpy()[:, 0].view(np.uint32), want[1].view(np.uint32))


# ------------------------------------------------------------------------------------------------
# 6: replicas through densify events
# ------------------------------------------------------------------------------------------------
def _thresholds(model, extent):
    """max_grad / min_opacity picked from the state so that the event clones, splits and prunes non-empty sets"""
    g = (model.xyz_gradient_accum / model.denom)[:, 0]
    g[g.isnan()] = 0.0
    nz = g[g > 0]
    max_grad = float(torch.quantile(nz, 0.8))
    ms = torch.exp(model._scaling.detach()).max(dim=1).values
    dense = model.percent_dense * extent
    clone = (g >= max_grad) & (ms <= dense)
    split = (g >= max_grad) & (ms > dense)
    op = torch.sigmoid(model._opacity.detach())[:, 0]
    min_op = float(torch.quantile(op, 0.05))
    prune = (op < min_op) & ~split
    return max_grad, min_op, int(clone.sum()), int(split.sum()), int(prune.sum())


def test_replicas_stay_identical_through_densify_events():
    world, P0, W, H, steps, events = 3, 20_000, 160, 120, 30, (10, 20)
    raw = make_scene(P0, sh_degree=3, seed=4, scale_mult=1.5)["raw"]
    models = [_Model(raw) for _ in range(world)]
    cams = make_cameras(12, W, H)
    settings = lambda cam, deg: _settings(cam, deg, (0.0, 0.0, 0.0), 1.0)  # noqa: E731
    gen = torch.Generator().manual_seed(5)
    targets = [torch.rand(3, H, W, generator=gen).cuda() for _ in cams]
    ms = torch.exp(models[0]._scaling.detach()).max(dim=1).values
    extent = float(torch.quantile(ms, 0.5)) / models[0].percent_dense   # half the Gaussians are "large": some split, some clone
    sim, cap, serial = None, 0, 0
    for s in range(steps):
        P = models[0]._xyz.shape[0]
        if sim is None or cap < P:             # the exchange grows its buffers as rasterizer._sparse_exchange does
            cap = int(P * 1.25)
            sim = None
            sim = _StatsSim(world, P, cap, nbufs=2, modes=("push",))
        k = s % 2
        serial += 1
        views = [cams[(s * world + r) % len(cams)] for r in range(world)]
        g2ds, radii_all = [], []
        for r, m in enumerate(models):         # rank r's pack of its own view, from its own replica
            leaves = [p.detach() for p in m.parameters()]
            rs = settings(views[r], 3)
            with torch.no_grad():
                _, _, R, color, radii, geom, binning, img, _ = _forward_raw_native(False, rs, *leaves)
            dpix = torch.sign(color - targets[(s * world + r) % len(cams)]) / float(3 * H * W)
            g2d = torch.empty((P, 3), device="cuda")
            _sparse_pack(sim.ranks["push"][r], k, rs, R, dpix, *leaves, radii, geom, binning, img, g2d, serial=serial)
            g2ds.append(g2d)
            radii_all.append(radii)
        for r, m in enumerate(models):         # after the barrier: the summed gradients, the statistics, the step
            leaves = [p.detach() for p in m.parameters()]
            g = [torch.empty(t.shape, device="cuda") for t in leaves]
            _sparse_accumulate(sim.ranks["push"][r], k, 3, world, leaves[0], leaves[2], g)
            filt = (radii_all[r] > 0).contiguous()
            densify.stats_exchanged(sim.ranks["push"][r], k, r, serial, world, g2ds[r], filt, m.xyz_gradient_accum, m.denom)
            m.max_radii2D[filt] = torch.max(m.max_radii2D[filt], radii_all[r][filt].float())   # per rank, never decides anything
            for p, gp in zip(m.parameters(), g):
                p.grad = gp
            m.optimizer.step()
            m.optimizer.zero_grad(set_to_none=True)
        if s + 1 in events:
            max_grad, min_op, nc, ns, npr = _thresholds(models[0], extent)
            assert nc > 0 and ns > 0 and npr > 0, f"step {s}: clone {nc} split {ns} prune {npr}"
            for m in models[1:]:
                assert _same(m.state()[:-1], models[0].state()[:-1]), f"step {s}: replicas differ before the event"
            rng = torch.cuda.get_rng_state()
            for m in models:
                torch.cuda.set_rng_state(rng)
                densify.densify_and_prune(m, max_grad, min_op, extent, None)
            ref = models[0].state()
            for r, m in enumerate(models[1:], 1):
                assert m._xyz.shape[0] == models[0]._xyz.shape[0], f"event at {s}: replica {r} P differs"
                assert _same(m.state(), ref), f"event at {s}: replica {r} differs from replica 0"
            assert models[0]._xyz.shape[0] != P
            print(f"\nevent after step {s}: P {P} -> {models[0]._xyz.shape[0]} (clone {nc}, split {ns}, prune >= {npr})")
    assert int(densify.error_word(torch.device("cuda")).item()) == 0


# ------------------------------------------------------------------------------------------------
# 7: bench size, once
# ------------------------------------------------------------------------------------------------
def test_stats_bench_size_world8():
    world, P, W, H = 8, 3_000_000, 1920, 1080
    raw = make_scene(P, sh_degree=3, seed=0)["raw"]
    pc = GaussianParams(raw, 3, "cuda", requires_grad=False)
    del raw
    leaves = [p.detach() for p in pc.parameters()]
    cams = make_cameras(16, W, H)[:world]
    settings = lambda cam, deg: _settings(cam, deg, (0.0, 0.0, 0.0), 1.0)  # noqa: E731
    gen = torch.Generator().manual_seed(1234)
    targets = [torch.rand(3, H, W, generator=gen) for _ in range(world)]
    sim = _StatsSim(world, P, P, nbufs=1, modes=("push",))
    g2d, radii = _pack_views(sim, 0, 77, leaves, 3, cams, settings,
                             lambda v, img: torch.sign(img - targets[v].cuda()) / float(3 * H * W), modes=("push",))
    filts = [(r > 0).contiguous() for r in radii]
    accum, denom = _seeded_stats(P, seed=99)
    outs = [_run_exchanged(sim.ranks["push"][r], 0, r, 77, world, g2d["push"][r], filts[r], accum, denom) for r in range(world)]
    assert int(densify.error_word(torch.device("cuda")).item()) == 0
    for a, d in outs[1:]:
        assert torch.equal(_bits(a), _bits(outs[0][0])) and torch.equal(_bits(d), _bits(outs[0][1]))
    ea, ed = _emulate(accum, denom, g2d["push"], filts)
    np.testing.assert_array_equal(outs[0][0].cpu().numpy()[:, 0].view(np.uint32), ea.view(np.uint32))
    np.testing.assert_array_equal(outs[0][1].cpu().numpy()[:, 0].view(np.uint32), ed.view(np.uint32))


# ------------------------------------------------------------------------------------------------
# 8: two real ranks (NCCL), skipped with one GPU
# ------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    from lightgaussian_b200 import parallel
    from lightgaussian_b200.model import TorchCamera, pipeline_params
    from lightgaussian_b200.renderer import render
    parallel.init_from_env("nccl")
    dev = torch.device("cuda", rank)
    torch.manual_seed(0)
    torch.cuda.manual_seed(0)
    raw = make_scene(20_000, sh_degree=3, seed=5, scale_mult=1.5)["raw"]
    with torch.cuda.device(dev):
        m = _Model(raw)
        cams = [TorchCamera(c, dev) for c in make_cameras(8, 160, 120)]
        bg = torch.zeros(3, device=dev)
        parallel.enable_gradient_exchange(world, densification=True)
        for s in range(6):
            cam = cams[(s * world + rank) % len(cams)]
            pkg = render(cam, m, pipeline_params(), bg)
            pkg["render"].abs().mean().backward()
            densify.add_densification_stats(m, pkg["viewspace_points"], pkg["visibility_filter"])
            m.optimizer.step()
            m.optimizer.zero_grad(set_to_none=True)
        ms = torch.exp(m._scaling.detach()).max(dim=1).values
        extent = float(torch.quantile(ms, 0.5)) / m.percent_dense
        g = (m.xyz_gradient_accum / m.denom)[:, 0]
        g[g.isnan()] = 0.0
        max_grad = float(torch.quantile(g[g > 0], 0.8))
        densify.densify_and_prune(m, max_grad, 0.005, extent, None)
        parallel.enable_gradient_exchange(1)
        torch.cuda.synchronize()
        torch.save([t.cpu() for t in m.state()], os.path.join(out, f"r{rank}.pt"))
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_identical_after_densify_event(tmp_path):
    import torch.multiprocessing as mp
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    a, b = (torch.load(os.path.join(tmp_path, f"r{r}.pt")) for r in range(world))
    assert a[0].shape[0] != 20_000, "the event changed nothing"
    assert _same(a, b), "the two ranks' models differ after the densify event"
