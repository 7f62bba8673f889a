"""The implicit GEMM's tile planner (``ddpo_igemm_plan``, host code in csrc/igemm.cu) over every igemm launch of an
SD2-base denoising step and PPO train pass: it picks an instantiated tile that fits the launch, from the shape alone,
and over each pass fills its waves better than the 128-row, N-only tile width it replaced.  (Single launches may trade
a little wave fill for a wider tile that re-reads fewer operands: 128 x 192 instead of 128 x 160 at N = 960.)"""
import pytest

import _igemm_census as ic

SMS = 132


def _share(m, n, plan):
    """the share of the CTA slots of the launch's waves that hold a tile"""
    bm, bn, ctas = plan[:3]
    tiles = -(-m // bm) * (n // bn)
    slots = SMS * ctas
    return tiles / (-(-tiles // slots) * slots)


@pytest.mark.parametrize("pass_name", sorted(ic.PASSES))
def test_plan_is_a_valid_tile_and_fills_waves_better(pass_name):
    from ddpo_b200 import ops
    flops = new = old = 0.0
    for call, count in ic.distinct(pass_name):
        m, n, k, geglu = ic.shape(call)
        plan = ops.igemm_plan(m, n, k, geglu)
        bm, bn, ctas, stages = plan
        assert bm in (64, 128) and n % bn == 0 and 1 <= ctas <= 4 and 2 <= stages <= 8, (call.test_id(), plan)
        assert bm * ctas >= 128, (call.test_id(), plan)           # at least two consumer warpgroups per SM
        if geglu:
            assert bn == ic.old_width(n, True)                    # the width the GEGLU weights are permuted for
        assert ops.igemm_plan(m, n, k, geglu, bm=bm, bn=bn) == plan
        before = ops.igemm_plan(m, n, k, geglu, bm=128, bn=ic.old_width(n, geglu))
        f = 2.0 * m * n * k * count
        flops, new, old = flops + f, new + f * _share(m, n, plan), old + f * _share(m, n, before)
    assert new / flops > old / flops + 0.02, (new / flops, old / flops)


def test_plan_depends_on_the_shape_only():
    """the same shape gets the same tile whatever was planned before, and every launch of a signature shares it"""
    from ddpo_b200 import ops
    shapes = sorted({ic.shape(c) for p in ic.PASSES for c in ic.launches(p)})
    first = [ops.igemm_plan(*s) for s in shapes]
    assert [ops.igemm_plan(*s) for s in reversed(shapes)] == first[::-1]


def test_overrides_force_the_tile_and_reject_what_does_not_exist():
    from ddpo_b200 import _lib, ops
    for bm in (64, 128):
        for bn in (32, 64, 96, 128, 160, 192):
            assert ops.igemm_plan(4096, 1920, 640, bm=bm, bn=bn)[:2] == (bm, bn)
    assert ops.igemm_plan(4096, 10240, 1280, True)[:2] == (128, 256)
    for bad in (dict(bm=64, bn=256), dict(bn=48), dict(bm=96), dict(bn=256)):
        with pytest.raises(_lib.DdpoError):
            ops.igemm_plan(4096, 1920, 640, **bad)
