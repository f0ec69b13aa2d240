"""The pointer tables of the sparse view-parallel exchange (rasterizer._exchange_tables), on the CPU: which slot of which rank's buffer a
rank packs its view into, and where its accumulate kernel reads each view from, in push and in pull mode."""
import pytest

from lightgaussian_b200.rasterizer import _exchange_tables

SLOT = 0x10000


def _bases(world):
    """two alternating buffers per rank at distinct, 256-byte aligned addresses: bases[k][q] = rank q's buffer k"""
    return [[0x7000_0000 + (2 * q + k) * world * SLOT for q in range(world)] for k in range(2)]


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_push_tables(world):
    bases = _bases(world)
    for r in range(world):
        pack, ptrs = _exchange_tables(bases, r, SLOT, push=True)
        assert len(pack) == len(ptrs) == 2
        for k in range(2):
            assert list(pack[k]) == [bases[k][q] + r * SLOT for q in range(world)]    # slot r of every rank's buffer
            assert list(ptrs[k]) == [bases[k][r] + v * SLOT for v in range(world)]    # every view from the local buffer


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_pull_tables(world):
    bases = _bases(world)
    for r in range(world):
        pack, ptrs = _exchange_tables(bases, r, SLOT, push=False)
        for k in range(2):
            assert list(pack[k]) == [bases[k][r] + r * SLOT]                          # own buffer, own slot, nowhere else
            assert list(ptrs[k]) == [bases[k][v] + v * SLOT for v in range(world)]    # view v from rank v's buffer


@pytest.mark.parametrize("world", [2, 3, 8])
def test_every_slot_written_by_exactly_one_rank_and_read_by_its_readers(world):
    """push: the N ranks' pack tables cover each (buffer, slot) exactly once, and every rank reads view v where rank v wrote it.
    pull: each rank writes one slot, and every rank reads view v from that slot."""
    bases = _bases(world)
    for push in (True, False):
        tabs = [_exchange_tables(bases, r, SLOT, push) for r in range(world)]
        for k in range(2):
            written = [p for r in range(world) for p in tabs[r][0][k]]
            assert len(written) == len(set(written)) == (world * world if push else world)
            for r in range(world):
                for v in range(world):
                    dst = list(tabs[v][0][k])
                    assert tabs[r][1][k][v] in dst
