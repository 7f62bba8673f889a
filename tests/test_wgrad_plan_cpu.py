"""The weight-gradient planner (``ddpo_wgrad_plan``, host code in csrc/wgrad.cu) over every wgrad call of an SD2-base,
SD1, TINY and SMALL train pass at batch 40: one launch of whole column tiles, a bounded workspace, a plan that depends
on the shape alone, and, weighted by FLOPs, fuller waves than the planner it replaced (a 256-wide launch plus a
remainder launch, over input channels padded to 128 per tap)."""
import ctypes

import pytest

import _wgrad_census as wc

SMS = 132


def _fill(rows, n, pb, launches):
    """useful multiply-adds over what the launches' waves could hold: launches = [(CTAs, BN, pixel blocks per CTA)] of
    128-row CTAs, one per SM"""
    held = sum(-(-ctas // SMS) * SMS * 128 * bn * per for ctas, bn, per in launches)
    return rows * n * pb / held


def _workspace_floats(m, c0, c1, n, taps):
    from ddpo_b200._lib import WgradArgs, lib
    a = WgradArgs()
    a.is_conv, a.m = 0, m
    a.c0, a.c1, a.n, a.taps = c0, c1, n, taps
    return int(lib().ddpo_wgrad_workspace_floats(ctypes.byref(a)))


@pytest.mark.parametrize("cfg_name", sorted(wc.CONFIGS))
def test_plan_is_one_launch_of_whole_tiles_and_fills_waves_better(cfg_name):
    from ddpo_b200 import ops
    flops = new = old = 0.0
    for call, count in wc.distinct(cfg_name):
        m, c0, c1, n, taps = wc.shape(call)
        bn, splits = ops.wgrad_plan(m, c0, n, c1, taps)
        pb, rows = -(-m // 64), taps * (c0 + c1)
        assert bn in (64, 128, 192, 256, 320) and n % bn == 0, (call.test_id(), bn)
        assert 1 <= splits <= max(1, pb // 8), (call.test_id(), splits)
        per = -(-pb // splits)
        assert -(-pb // per) == splits, "no empty pixel split"
        need = _workspace_floats(m, c0, c1, n, taps)
        assert need == (splits * rows * n if splits > 1 else 0) and need <= 14745600, (call.test_id(), need)
        assert ops.wgrad_plan(m, c0, n, c1, taps, bn=bn, splits=splits) == (bn, splits)
        old_s, old_launches = wc.old_plan(m, c0, c1, n, taps)
        old_per = -(-pb // old_s)
        old_widths = ([256] if n >= 256 else []) + ([n % 256] if n % 256 else [])
        f = 2.0 * m * n * rows * count
        flops += f
        new += f * _fill(rows, n, pb, [(-(-rows // 128) * (n // bn) * splits, bn, per)])
        old += f * _fill(rows, n, pb, [(c, w, old_per) for c, w in zip(old_launches, old_widths)])
    assert new / flops > old / flops + 0.05, (cfg_name, new / flops, old / flops)


def test_plan_depends_on_the_shape_only():
    """the same shape gets the same plan whatever was planned before, and every call of a signature shares it"""
    from ddpo_b200 import ops
    shapes = sorted({wc.shape(c) for cfg in wc.CONFIGS for c in wc.calls(cfg)})
    first = [ops.wgrad_plan(m, c0, n, c1, taps) for m, c0, c1, n, taps in shapes]
    assert [ops.wgrad_plan(m, c0, n, c1, taps) for m, c0, c1, n, taps in reversed(shapes)] == first[::-1]


def test_overrides_force_the_plan_and_reject_what_does_not_exist():
    from ddpo_b200 import _lib, ops
    for bn in (64, 128, 192, 256, 320):
        assert ops.wgrad_plan(40 * 4096, 320, 3840, taps=9, bn=bn)[0] == bn     # 3840 = lcm of the widths
    assert ops.wgrad_plan(8192, 320, 320, splits=7)[1] == 7
    for bad in (dict(bn=96), dict(bn=256), dict(splits=129)):
        with pytest.raises(_lib.DdpoError):
            ops.wgrad_plan(8192, 320, 320, **bad)
    with pytest.raises(_lib.DdpoError):
        ops.wgrad_plan(8192, 96, 320)          # input channels in whole 64-channel units
