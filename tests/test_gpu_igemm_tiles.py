"""The implicit GEMM's output tile (BM x BN) is a scheduling choice, never an arithmetic one: every instantiated tile
that divides N gives the same bits as the 128-row tile at the width the library used before tiles were planned per
shape (outputs, GEGLU pre-activations and GroupNorm slab statistics), at U-Net shapes of SD2-base and SD1.x (same
convolution channels; the cross-attention context width differs).  Run on an H100: ``pytest -m gpu``."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
WIDTHS = (32, 64, 96, 128, 160, 192, 256)


def bf(x):
    return x.to(torch.bfloat16)


def old_width(n, geglu=False):
    """the tile width chosen from N alone, with 128-row tiles, before the planner"""
    for w in ((256, 192, 128, 64) if geglu else (128, 160, 192, 96, 64, 32)):
        if n % w == 0:
            return w


def tiles(m, n, k, geglu=False, bn=0):
    """every (BM, BN) the library has for this shape: the planned one first, then each override that resolves"""
    from ddpo_b200 import _lib, ops
    out = [(0, 0)]
    for bm in (64, 128):
        for w in ((bn,) if bn else WIDTHS):
            if n % w:
                continue
            try:
                plan = ops.igemm_plan(m, n, k, geglu, bm=bm, bn=w)
            except _lib.DdpoError:
                continue
            assert plan[:2] == (bm, w)
            out.append((bm, w))
    return out


def _prep_w(w_kn, geglu_bn=0):
    from ddpo_b200 import ops
    k, n = w_kn.shape
    dst = torch.empty(n, k, dtype=torch.bfloat16, device=DEV)
    ops.prep_weight(w_kn.contiguous(), dst, k, n, geglu_bn=geglu_bn)
    return dst


def _same(runs):
    ref = runs[0]
    for tile, outs in runs[1:]:
        for a, b in zip(ref[1], outs):
            if a is not None:
                assert torch.isfinite(a.float()).all() and torch.equal(a, b), (ref[0], tile)


# (batch, output grid, c0, c1, n, taps, stride): the U-Net's convolutions at every level, skip concats, the stride-2
# down-samples and 1x1 shortcuts, at batches that leave ragged last waves
CONVS = [(2, 64, 320, 0, 320, 9, 1), (3, 32, 640, 320, 640, 9, 1), (2, 16, 1280, 640, 1280, 9, 1),
         (5, 8, 1280, 1280, 1280, 9, 1), (2, 32, 320, 0, 320, 9, 2), (3, 8, 1280, 0, 1280, 9, 2),
         (2, 32, 640, 320, 640, 1, 1), (1, 4, 64, 0, 96, 9, 1)]


@pytest.mark.parametrize("b,h,c0,c1,n,taps,stride", CONVS)
def test_conv_every_tile_is_bit_identical(b, h, c0, c1, n, taps, stride):
    """fp32 output with bias, time-embedding row vector, residual and slab statistics; bf16 output; accumulate"""
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(b * 1000 + h + n)
    hi = h * stride
    m, cin = b * h * h, c0 + c1
    x0 = bf(torch.randn(b, hi, hi, c0, generator=g)).to(DEV)
    x1 = bf(torch.randn(b, hi, hi, c1, generator=g)).to(DEV) if c1 else None
    w = (torch.randn(taps * cin, n, generator=g) / math.sqrt(taps * cin)).to(DEV)
    bias = torch.randn(n, generator=g).to(DEV)
    res = torch.randn(m, n, generator=g).to(DEV)
    tv = torch.randn(b, n, generator=g).to(DEV)
    init = torch.randn(m, n, generator=g).to(DEV)
    wt = _prep_w(w)
    k = taps * cin
    order = [(128, old_width(n))] + [t for t in tiles(m, n, k) if t != (128, old_width(n))]
    runs = []
    for bm, bn in order:
        out = torch.zeros(m, n, device=DEV)
        ob = torch.zeros(m, n, dtype=torch.bfloat16, device=DEV)
        acc = init.clone()
        st = torch.full(ops.gn_stats_shape(m, n), float("nan"), device=DEV)
        kw = dict(a0=x0, a1=x1, wt=wt, n=n, c0=c0, c1=c1, conv=(b, h, h), taps=taps, stride=stride, bm=bm, bn=bn)
        ops.igemm(**kw, bias=bias, rowvec=tv, rows_per_sample=h * h, rowvec_ld=n, residual=res, out_f32=out, gn_stats=st)
        ops.igemm(**kw, bias=bias, out_bf16=ob)
        ops.igemm(**kw, out_f32=acc, accumulate=True)
        runs.append(((bm, bn), (out, st, ob, acc)))
    torch.cuda.synchronize()
    assert len(runs) >= 3
    _same(runs)


# (m, k, n): projections and feed-forward outputs at token counts of both models (77-token contexts, SD1's 768-wide and
# SD2's 1024-wide), ragged M
LINEARS = [(154, 1024, 640), (154, 768, 1280), (4096 + 77, 320, 320), (1000, 2560, 1280), (2048, 640, 1920)]


@pytest.mark.parametrize("m,k,n", LINEARS)
def test_linear_every_tile_is_bit_identical(m, k, n):
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(m + k + n)
    a = bf(torch.randn(m, k, generator=g)).to(DEV)
    w = (torch.randn(k, n, generator=g) / math.sqrt(k)).to(DEV)
    bias = torch.randn(n, generator=g).to(DEV)
    res = torch.randn(m, n, generator=g).to(DEV)
    wt = _prep_w(w)
    order = [(128, old_width(n))] + [t for t in tiles(m, n, k) if t != (128, old_width(n))]
    runs = []
    for bm, bn in order:
        out = torch.zeros(m, n, device=DEV)
        ob = torch.zeros(m, n, dtype=torch.bfloat16, device=DEV)
        st = torch.full(ops.gn_stats_shape(m, n), float("nan"), device=DEV)
        ops.igemm(a0=a, wt=wt, n=n, c0=k, m=m, bias=bias, residual=res, out_f32=out, out_bf16=ob, gn_stats=st, bm=bm, bn=bn)
        runs.append(((bm, bn), (out, st, ob)))
    torch.cuda.synchronize()
    _same(runs)
    ref = a.float() @ bf(w).float() + bias + res
    assert (runs[0][1][0] - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("m,k", [(1000, 320), (4096 + 77, 640), (2 * 64, 1280)])
@pytest.mark.parametrize("gbn", [256, 128, 64])
def test_geglu_both_tile_heights_are_bit_identical(m, k, gbn):
    """GEGLU keeps the width its weights were permuted for; every height at that width gives the same activations and
    pre-activations"""
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(m + k + gbn)
    n = 8 * k
    a = bf(torch.randn(m, k, generator=g)).to(DEV)
    w = (torch.randn(k, n, generator=g) / math.sqrt(k)).to(DEV)
    b = torch.randn(n, generator=g).to(DEV)
    wt = _prep_w(w, geglu_bn=gbn)
    bp = torch.empty_like(b)
    ops.permute_geglu_bias(b, bp, n, gbn)
    runs = []
    for bm, bn in [(128, gbn)] + [t for t in tiles(m, n, k, geglu=True, bn=gbn) if t != (128, gbn)]:
        o = torch.full((m, n // 2), 3.0, dtype=torch.bfloat16, device=DEV)
        aux = torch.full((m, n), 5.0, dtype=torch.bfloat16, device=DEV)
        ops.igemm(a0=a, wt=wt, n=n, c0=k, m=m, bias=bp, out_bf16=o, geglu=True, aux_bf16=aux, bm=bm, bn=bn or gbn)
        runs.append(((bm, bn), (o, aux)))
    torch.cuda.synchronize()
    assert len(runs) >= (2 if gbn == 256 else 3)
    _same(runs)
