"""Default blend backward (CPU check of the built library): a flush adds each (warp, Gaussian) row of nine moment sums to its 48-byte
accumulator record with two 16-byte vector reductions (words 0-3 and 4-7) and one scalar reduction (word 8), not with nine scalar
ones.  Each SASS reduction instruction sends one L2 operation per active lane, so this is what keeps the L2 atomic traffic at three
operations per pair."""
import re

from tests.test_deterministic_sass import _find, sass  # noqa: F401  (module fixture: the library's SASS by kernel name)

REDG_F32 = re.compile(r"\bREDG\.E\.ADD\.(F32x4|F32)\.")


def test_blend_backward_flush_uses_vector_reductions(sass):  # noqa: F811
    for name in _find(sass, "blend_backward_ring_kernelILb0E"):
        ops = REDG_F32.findall(sass[name])
        v4, scalar = ops.count("F32x4"), ops.count("F32")
        assert v4 >= 2, f"{name}: no REDG.E.ADD.F32x4 pair in the flush ({ops})"
        # every flush site issues two vector reductions, so this allows one scalar reduction per site
        assert scalar <= v4 // 2, f"{name}: {scalar} scalar F32 reductions for {v4} vector ones"
