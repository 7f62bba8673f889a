"""The weight-gradient GEMM at every plan it can run: each column-tile width and split count forced through the
overrides, rows in 64-channel units that straddle a tap or a source boundary, a half-empty last CTA row, stride 2 and
column slices of dY.  Each case accumulates into a flat-buffer slot with a non-zero prior, is checked against float64
with the bound of test_param_grad_layers.py, writes nothing past its slot or workspace, and gives the same bits twice."""
import ctypes

import pytest
import torch
from _layer_check import BF16, FlatSlot, check_sum, rnd
from test_param_grad_layers import _OwnWorkspace, _wgrad_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _need(conv, m, c0, c1, n, taps, stride, bn, splits):
    from ddpo_b200._lib import WgradArgs, lib
    a = WgradArgs()
    if conv is not None:
        a.is_conv, a.batch, a.h, a.w = 1, *conv
    else:
        a.is_conv, a.m = 0, m
    a.c0, a.c1, a.n, a.taps, a.conv_stride = c0, c1, n, taps, stride
    a.bn_override, a.splits_override = bn, splits
    return int(lib().ddpo_wgrad_workspace_floats(ctypes.byref(a)))


def _run(calls, slots, plan):
    """the wgrad ``calls`` into their slots, twice from the same prior; returns the first run's results"""
    from ddpo_b200 import ops
    outs = []
    for _ in range(2):
        for s in slots:
            s.view.copy_(s.prior())
        with _OwnWorkspace(ops, DEV, _need(*plan)) as ws:
            for kw, s in zip(calls, slots):
                ops.wgrad(dw=s.view, **kw)
            torch.cuda.synchronize()
        ws.check("wgrad")
        for s in slots:
            s.check("wgrad")
        outs.append([s.view.clone() for s in slots])
    for a, b in zip(*outs):
        assert torch.equal(a, b), "two runs from the same prior differ"
    return outs[0]


# (b, h, w of dY, c0, c1, n, taps, stride, bn, splits); bn / splits 0 = planned
CASES = [
    # every width, one and several splits (c_in = 320: 5 units per tap, so CTA rows straddle taps; 45 units in all)
    *[(2, 16, 16, 320, 0, 2 * bn, 9, 1, bn, s) for bn in (64, 128, 192, 256, 320) for s in (1, 3)],
    # straddling units at the planned widths: c_in = 192 (3 units per tap), 960 (15), and one 64-channel unit
    (2, 16, 16, 192, 0, 128, 9, 1, 0, 0), (2, 8, 8, 960, 0, 640, 9, 1, 0, 0), (4, 16, 16, 64, 0, 320, 9, 1, 320, 2),
    # two sources: the source boundary falls inside a unit pair, in both orders, with 3x3 and 1x1 taps
    (2, 16, 16, 320, 640, 320, 9, 1, 0, 0), (2, 16, 16, 640, 320, 320, 9, 1, 320, 1),
    (2, 16, 16, 320, 640, 640, 1, 1, 128, 2), (2, 16, 16, 640, 320, 320, 1, 1, 0, 0),
    # stride 2 (dY is h x w, X is 2h x 2w)
    (2, 16, 16, 320, 0, 320, 9, 2, 0, 0), (2, 16, 16, 640, 0, 640, 9, 2, 320, 4),
]


@pytest.mark.parametrize("b,h,w,c0,c1,n,taps,stride,bn,splits", CASES)
def test_wgrad_forced_and_straddling_plans(b, h, w, c0, c1, n, taps, stride, bn, splits):
    g = torch.Generator().manual_seed(211 + c0 + 3 * c1 + n + bn + splits + stride)
    hi, wi = h * stride, w * stride
    x0 = rnd(g, b * hi * wi, c0).to(BF16).to(DEV)
    x1 = rnd(g, b * hi * wi, c1).to(BF16).to(DEV) if c1 else None
    dy = rnd(g, b * h * w, n).to(BF16).to(DEV)
    rows = taps * (c0 + c1)
    slot = FlatSlot(rows, n, DEV, rnd(g, rows, n, scale=float(b * h * w) ** 0.5), after=128 * n)
    kw = dict(dy=dy, n=n, x0=x0, c0=c0, x1=x1, c1=c1, conv=(b, h, w), taps=taps, stride=stride, bn=bn, splits=splits)
    out = _run([kw], [slot], ((b, h, w), None, c0, c1, n, taps, stride, bn, splits))[0]
    x = x0 if x1 is None else torch.cat([x0, x1], 1)
    ref, terms = _wgrad_ref(x, dy, (b, h, w), taps, stride)
    check_sum("dw", out, ref, terms, old=slot.prior())


@pytest.mark.parametrize("bn,splits", [(320, 0), (64, 5), (192, 1), (0, 0)])
def test_wgrad_qkv_column_slices(bn, splits):
    """to_q / to_k / to_v: dY is a column slice of one [m, 3C] gradient with pitch 3C (C = 960 takes every width but 256)"""
    g = torch.Generator().manual_seed(223 + bn + splits)
    c, m = 960, 2 * 1024
    x = rnd(g, m, c).to(BF16).to(DEV)
    dqkv = rnd(g, m, 3 * c).to(BF16).to(DEV)
    slots = [FlatSlot(c, c, DEV, rnd(g, c, c, scale=m ** 0.5), after=128 * c, seed=70 + i) for i in range(3)]
    calls = [dict(dy=dqkv[:, i * c:], ldy=3 * c, n=c, x0=x, c0=c, m=m, bn=bn, splits=splits) for i in range(3)]
    outs = _run(calls, slots, (None, m, c, 0, c, 1, 1, bn, splits))
    ref, terms = _wgrad_ref(x, dqkv, None)
    for i, out in enumerate(outs):
        cols = slice(i * c, (i + 1) * c)
        check_sum(f"slice {i}", out, ref[:, cols], terms[:, cols], old=slots[i].prior())


def test_wgrad_kv_slices_of_ragged_context():
    """attn2 to_k / to_v: X is the text context, m = b * 77 rows (a ragged last pixel block), dY slices of pitch 2C"""
    g = torch.Generator().manual_seed(227)
    c, dctx, m = 320, 1024, 2 * 77
    ctx = rnd(g, m, dctx).to(BF16).to(DEV)
    dkv = rnd(g, m, 2 * c).to(BF16).to(DEV)
    slots = [FlatSlot(dctx, c, DEV, rnd(g, dctx, c, scale=m ** 0.5), after=128 * c, seed=60 + i) for i in range(2)]
    calls = [dict(dy=dkv[:, i * c:], ldy=2 * c, n=c, x0=ctx, c0=dctx, m=m) for i in range(2)]
    outs = _run(calls, slots, (None, m, dctx, 0, c, 1, 1, 0, 0))
    ref, terms = _wgrad_ref(ctx, dkv, None)
    for i, out in enumerate(outs):
        cols = slice(i * c, (i + 1) * c)
        check_sum(f"slice {i}", out, ref[:, cols], terms[:, cols], old=slots[i].prior())
