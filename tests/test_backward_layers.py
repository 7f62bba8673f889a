"""The U-Net backward pass (ddpo_b200/unet.py, ``UNet.backward``) layer by layer: every CUDA entry point of the train pass,
called with the arguments, pitches and compositions unet.py uses, against a float64 torch reference fed the same
bf16-rounded operands the kernel sees.  The whole-model gradient tests (test_gpu_training.py, test_gpu_sd2_parity.py)
allow up to 0.2 of relative error on a parameter tensor, enough to hide a defect confined to one layer (a wrong tap on
a border pixel, a dropped ``accumulate``); these checks are per layer and tight.

Conventions:
- error bounds: a max-abs error relative to max|ref| AND a relative L2 error (L2 alone hides border-pixel errors);
  reductions (column sums, dscale / dbias, dense dW / db / dx) are bounded per element by a multiple of the sum of the
  absolute values of the summed terms, so that cancellation cannot make the bound meaningless;
- exact operations (weight layout, zero dilation, the bf16 copy of a gradient, copies) are compared bit for bit;
- every output lives inside a larger buffer (extra columns past the pitch where the op takes a pitch, extra rows after
  the last row) whose outside part must come back unchanged: a write past the end lands in memory the test owns.

The layer-shaped checks also run at small shapes on the torch-CPU emulation of the ops (tests/_cpu_ops_emulator.py)
that the CPU dry runs of the train path depend on; the CUDA variants carry the ``gpu`` mark.

Every check stores its measured errors as test properties (``pytest --junitxml=...`` writes them out), so that the
margins of the bounds below are on record.
"""
import pytest
import torch
import torch.nn.functional as F
from _layer_check import (ATT_L2, ATT_MAX, BF16, BF16_L2, BF16_MAX, F32, F32_L2, F32_MAX, F64, SUM_TOL, Backend,
                          Guarded, _backend_params, _current_node, _record, check_close, check_sum, rnd)  # noqa: F401


def hwio_to_oihw(w):
    """Flax conv kernel [kh, kw, cin, cout] -> torch [cout, cin, kh, kw]"""
    return w.permute(3, 2, 0, 1)


def nhwc(t, b, h, w):
    return t.reshape(b, h, w, -1).permute(0, 3, 1, 2)


def rows_of(t):
    """NCHW -> [b*h*w, c]"""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def dgrad_weight(be, w, taps, cin, n):
    """the dgrad-layout bf16 weight unet.py keeps per layer (UNet._refresh_dgrad_weights)"""
    wd = torch.empty(cin, taps * n, dtype=BF16, device=be.dev)
    be.ops.prep_weight_dgrad(w.to(be.dev), wd, taps, cin, n)
    return wd


# ------------------------------------------------------------------------- 1. data-gradient convolutions ------
@pytest.mark.parametrize("backend,taps,k,n,ld,col", _backend_params(
    [(9, 128, 64, 0, 0), (9, 192, 96, 0, 0), (1, 64, 64, 256, 64), (1, 320, 320, 960, 0), (1, 320, 320, 960, 640),
     (9, 1920, 640, 0, 0), (1, 128, 96, 512, 96)]))
def test_prep_weight_dgrad_layout(backend, taps, k, n, ld, col):
    """dst[k, col + tap*n + j] = bf16(w)[rotated 180 degrees][tap, k, j]; other columns keep what they held"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(taps * 1000 + k + n)
    ks = 3 if taps == 9 else 1
    w = rnd(g, ks, ks, k, n, scale=0.05)
    pitch = ld or taps * n
    dst = Guarded(k, pitch, BF16, be.dev, extra_rows=2)
    be.ops.prep_weight_dgrad(w.reshape(taps, k, n).to(be.dev), dst.view, taps, k, n, ld_dst=ld, col_offset=col)
    be.sync()
    ref = w.to(BF16).flip(0, 1).permute(2, 0, 1, 3).reshape(k, taps * n)   # [k, (ky', kx', j)] with ky' = 2 - ky
    assert torch.equal(dst.view[:, col:col + taps * n].cpu(), ref)
    outside = torch.ones(k, pitch, dtype=torch.bool)
    outside[:, col:col + taps * n] = False
    assert torch.equal(dst.view.cpu()[outside], dst.snapshot[:k].cpu()[outside]), "columns outside the written range"
    dst.check("prep_weight_dgrad")


def _conv_dgrad_ref(dy_b, w, b, h, w_, cin, stride=1, padding=1):
    """float64 input gradient of y = conv2d(x, w) for the bf16 operands (dy_b NHWC rows, w HWIO)"""
    dev = dy_b.device
    ho, wo = h // stride, w_ // stride
    return torch.nn.grad.conv2d_input((b, cin, h, w_), hwio_to_oihw(w.to(BF16).double()).to(dev),
                                      nhwc(dy_b.double(), b, ho, wo), stride=stride, padding=padding)


@pytest.mark.parametrize("out_dtype", ["f32", "bf16"])
@pytest.mark.parametrize("backend,b,h,w,cout,cin", _backend_params(
    [(2, 8, 16, 64, 128), (1, 4, 4, 128, 192)],
    [(2, 8, 8, 1280, 2560), (2, 16, 16, 1280, 1920), (2, 32, 32, 640, 960), (2, 64, 64, 320, 640),
     (2, 16, 32, 320, 640)]))
def test_conv3x3_dgrad(backend, b, h, w, cout, cin, out_dtype):
    """resnet conv1 dgrad (unet.py:631): N = cin of a two-source resnet, K = 9 * cout"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(b * h * w + cout + cin)
    m = b * h * w
    wt = rnd(g, 3, 3, cin, cout, scale=(9 * cin) ** -0.5)
    dyb = rnd(g, m, cout).to(BF16).to(be.dev)
    wd = dgrad_weight(be, wt, 9, cin, cout)
    dt = F32 if out_dtype == "f32" else BF16
    out = Guarded(m, cin, dt, be.dev, extra_cols=be.pad)
    kw = {"out_f32": out.arg} if dt == F32 else {"out_bf16": out.arg}
    be.ops.igemm(a0=dyb, wt=wd, n=cin, c0=cout, conv=(b, h, w), taps=9, ld_out=out.ld, **kw)
    be.sync()
    ref = rows_of(_conv_dgrad_ref(dyb, wt, b, h, w, cin))
    tol = (F32_MAX, F32_L2) if dt == F32 else (BF16_MAX, BF16_L2)
    check_close("dx", out.view, ref, *tol)
    out.check("conv3x3 dgrad")


@pytest.mark.parametrize("backend,b,h,w,cout,cin", _backend_params(
    [(2, 8, 16, 64, 128)], [(2, 16, 16, 1280, 2560), (2, 64, 32, 320, 640), (2, 32, 32, 640, 960)]))
def test_conv1x1_shortcut_dgrad(backend, b, h, w, cout, cin):
    """conv_shortcut dgrad (unet.py:637): fp32 output that the norm1 backward then accumulates into"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(7 + cin)
    m = b * h * w
    wt = rnd(g, 1, 1, cin, cout, scale=cin ** -0.5)
    dyb = rnd(g, m, cout).to(BF16).to(be.dev)
    wd = dgrad_weight(be, wt, 1, cin, cout)
    out = Guarded(m, cin, F32, be.dev, extra_cols=be.pad)
    be.ops.igemm(a0=dyb, wt=wd, n=cin, c0=cout, conv=(b, h, w), taps=1, out_f32=out.arg, ld_out=out.ld)
    be.sync()
    ref = rows_of(_conv_dgrad_ref(dyb, wt, b, h, w, cin, padding=0))
    check_close("dx", out.view, ref, F32_MAX, F32_L2)
    out.check("conv1x1 dgrad")


@pytest.mark.parametrize("backend,b,h,w,c", _backend_params([(2, 4, 8, 64), (1, 2, 2, 128)], [(2, 32, 32, 320), (2, 8, 16, 1280)]))
def test_dilate2x_bf16_exact(backend, b, h, w, c):
    """y[b, 2i, 2j] = bf16(x[b, i, j]), zeros at every odd row or column"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(11)
    x = rnd(g, b * h * w, c)
    y = Guarded(b * 4 * h * w, c, BF16, be.dev)
    be.ops.dilate2x_bf16(x.to(be.dev), y.view, b, h, w, c)
    be.sync()
    ref = torch.zeros(b, 2 * h, 2 * w, c, dtype=BF16)
    ref[:, ::2, ::2] = x.reshape(b, h, w, c).to(BF16)
    assert torch.equal(y.view.cpu(), ref.reshape(-1, c))
    y.check("dilate2x")


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("backend,b,h,w,c", _backend_params(
    [(2, 8, 16, 64)], [(2, 64, 64, 320), (2, 32, 32, 640), (2, 16, 16, 1280), (2, 32, 64, 320)]))
def test_downsample_dgrad(backend, b, h, w, c, accumulate):
    """stride-2 conv dgrad as unet.py:551-559: zero-dilate dy, then a stride-1 3x3 igemm with the rotated kernel,
    accumulated into the gradient the stream tensor already has (or into a fresh one)"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(13 + c + h)
    m, mo = b * h * w, b * (h // 2) * (w // 2)
    wt = rnd(g, 3, 3, c, c, scale=(9 * c) ** -0.5)
    dy = rnd(g, mo, c)                                      # fp32 gradient of the downsampler output
    old = rnd(g, m, c, scale=0.5)
    wd = dgrad_weight(be, wt, 9, c, c)
    dil = torch.empty(m, c, dtype=BF16, device=be.dev)
    be.ops.dilate2x_bf16(dy.to(be.dev), dil, b, h // 2, w // 2, c)
    out = Guarded(m, c, F32, be.dev, extra_cols=be.pad, init=old if accumulate else None)
    be.ops.igemm(a0=dil, wt=wd, n=c, c0=c, conv=(b, h, w), taps=9, out_f32=out.arg, ld_out=out.ld,
                 accumulate=accumulate)
    be.sync()
    ref = rows_of(_conv_dgrad_ref(dy.to(BF16).to(be.dev), wt, b, h, w, c, stride=2))
    got = out.view.double() - (old.to(be.dev).double() if accumulate else 0)
    check_close("dx", got, ref, F32_MAX, F32_L2)
    out.check("downsample dgrad")


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("backend,b,h,w,c", _backend_params(
    [(2, 4, 8, 64)], [(2, 8, 8, 1280), (2, 16, 16, 1280), (2, 32, 32, 640), (2, 16, 32, 320)]))
def test_upsample_block_dgrad(backend, b, h, w, c, accumulate):
    """upsampler (unet.py:534-541): y = conv3x3(nearest2x(x)); conv dgrad at (2h, 2w), then upsample2x_bwd into a fresh
    gradient or on top of the one x already has"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(17 + c + h)
    m, m2 = b * h * w, b * 4 * h * w
    wt = rnd(g, 3, 3, c, c, scale=(9 * c) ** -0.5)
    dyb = rnd(g, m2, c).to(BF16).to(be.dev)
    old = rnd(g, m, c, scale=0.5)
    wd = dgrad_weight(be, wt, 9, c, c)
    d_up = Guarded(m2, c, F32, be.dev, extra_cols=be.pad)
    be.ops.igemm(a0=dyb, wt=wd, n=c, c0=c, conv=(b, 2 * h, 2 * w), taps=9, out_f32=d_up.arg, ld_out=d_up.ld)
    dx = Guarded(m, c, F32, be.dev, init=old if accumulate else None)
    be.ops.upsample2x_bwd(d_up.view.contiguous(), dx.view, b, h, w, c, accumulate=accumulate)
    be.sync()
    x = torch.zeros(b, c, h, w, dtype=F64, device=be.dev, requires_grad=True)
    y = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), hwio_to_oihw(wt.to(BF16).double()).to(be.dev),
                 padding=1)
    y.backward(nhwc(dyb.double(), b, 2 * h, 2 * w))
    check_close("d_up", d_up.view, rows_of(_conv_dgrad_ref(dyb, wt, b, 2 * h, 2 * w, c)), F32_MAX, F32_L2)
    got = dx.view.double() - (old.to(be.dev).double() if accumulate else 0)
    check_close("dx", got, rows_of(x.grad), F32_MAX, F32_L2)
    d_up.check("upsampler conv dgrad")
    dx.check("upsample2x_bwd")


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("backend,b,h,w,c", _backend_params([(2, 4, 8, 4), (1, 2, 2, 8)], [(2, 32, 32, 640), (40, 16, 32, 320)]))
def test_upsample2x_bwd(backend, b, h, w, c, accumulate):
    """dx[b, i, j] (+)= sum of the 2x2 block dy[b, 2i:2i+2, 2j:2j+2]"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(19 + c)
    dy = rnd(g, b, 2 * h, 2 * w, c)
    old = rnd(g, b * h * w, c)
    dx = Guarded(b * h * w, c, F32, be.dev, init=old if accumulate else None)
    be.ops.upsample2x_bwd(dy.to(be.dev).reshape(-1, c), dx.view, b, h, w, c, accumulate=accumulate)
    be.sync()
    blocks = dy.double().reshape(b, h, 2, w, 2, c)
    ref = blocks.sum(dim=(2, 4)).reshape(-1, c)
    terms = blocks.abs().sum(dim=(2, 4)).reshape(-1, c)
    check_sum("dx", dx.view.cpu(), ref, terms, old=old if accumulate else None)
    dx.check("upsample2x_bwd")


@pytest.mark.parametrize("backend,m,c", _backend_params([(96, 64), (100, 128)], [(8192, 320), (512, 1280), (2 * 77 * 16, 640)]))
def test_self_attention_qkv_dgrad(backend, m, c):
    """input gradient of the fused q/k/v projection (unet.py:184, 732): ONE GEMM over K = 3C, the weight assembled by
    three prep_weight_dgrad calls into column slots of a [C, 3C] buffer"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(23 + c)
    ws = [rnd(g, c, c, scale=c ** -0.5) for _ in range(3)]
    wd = torch.empty(c, 3 * c, dtype=BF16, device=be.dev)
    for i, w in enumerate(ws):
        be.ops.prep_weight_dgrad(w.to(be.dev), wd, 1, c, c, ld_dst=3 * c, col_offset=i * c)
    dqkv = rnd(g, m, 3 * c).to(BF16).to(be.dev)
    out = Guarded(m, c, BF16, be.dev, extra_cols=be.pad)
    be.ops.igemm(a0=dqkv, c0=3 * c, wt=wd, n=c, m=m, out_bf16=out.arg, ld_out=out.ld)
    be.sync()
    d = dqkv.double()
    ref = sum(d[:, i * c:(i + 1) * c] @ ws[i].to(BF16).double().to(be.dev).t() for i in range(3))
    check_close("d_ln", out.view, ref, BF16_MAX, BF16_L2)
    out.check("qkv dgrad")


@pytest.mark.parametrize("backend,m,c", _backend_params([(100, 64)], [(2048, 640), (128, 1280), (8192, 320)]))
def test_geglu_projection_dgrad(backend, m, c):
    """GEGLU backward then the proj dgrad (unet.py:690-696): geglu_bwd reads the tile-interleaved pre-activation and
    writes the gradient in the plain [lin(4C) | gate(4C)] order of the Flax kernel, over which the dgrad runs K = 8C"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(29 + c)
    n = 8 * c
    lin, gate = rnd(g, m, 4 * c).to(BF16), rnd(g, m, 4 * c).to(BF16)
    pre = torch.empty(m, n, dtype=BF16)
    for t in range(n // 256):
        pre[:, t * 256:t * 256 + 128] = lin[:, t * 128:(t + 1) * 128]
        pre[:, t * 256 + 128:(t + 1) * 256] = gate[:, t * 128:(t + 1) * 128]
    dff = rnd(g, m, 4 * c).to(BF16)
    w = rnd(g, c, n, scale=n ** -0.5)                       # Flax proj kernel [C, 8C]
    d_pre = torch.empty(m, n, dtype=BF16, device=be.dev)
    be.ops.geglu_bwd(pre.to(be.dev), dff.to(be.dev), d_pre, m, n, 256)
    wd = dgrad_weight(be, w, 1, c, n)
    out = Guarded(m, c, BF16, be.dev, extra_cols=be.pad)
    be.ops.igemm(a0=d_pre, wt=wd, n=c, c0=n, m=m, out_bf16=out.arg, ld_out=out.ld)
    be.sync()
    lr, gr = lin.double().requires_grad_(True), gate.double().requires_grad_(True)
    (lr * F.gelu(gr, approximate="tanh")).backward(dff.double())
    check_close("d_pre", d_pre.cpu(), torch.cat([lr.grad, gr.grad], 1), BF16_MAX, BF16_L2)
    ref = d_pre.double() @ w.to(BF16).double().to(be.dev).t()   # the dgrad on the bf16 gradient the kernel wrote
    check_close("d_ln", out.view, ref, BF16_MAX, BF16_L2)
    out.check("geglu proj dgrad")


@pytest.mark.parametrize("out_dtype", ["f32", "bf16"])
@pytest.mark.parametrize("backend,m,c", _backend_params([(100, 128)], [(8192, 320), (130, 1280), (2048, 640)]))
def test_linear_dgrad(backend, m, c, out_dtype):
    """plain C -> C linear dgrad (proj_out / proj_in / to_out / to_q, unet.py:679, 705, 716, 740)"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(31 + c)
    w = rnd(g, c, c, scale=c ** -0.5)
    dyb = rnd(g, m, c).to(BF16).to(be.dev)
    wd = dgrad_weight(be, w, 1, c, c)
    dt = F32 if out_dtype == "f32" else BF16
    out = Guarded(m, c, dt, be.dev, extra_cols=be.pad)
    kw = {"out_f32": out.arg} if dt == F32 else {"out_bf16": out.arg}
    be.ops.igemm(a0=dyb, wt=wd, n=c, c0=c, m=m, ld_out=out.ld, **kw)
    be.sync()
    ref = dyb.double() @ w.to(BF16).double().to(be.dev).t()
    check_close("dx", out.view, ref, *((F32_MAX, F32_L2) if dt == F32 else (BF16_MAX, BF16_L2)))
    out.check("linear dgrad")


# --------------------------------------------------------------------------- 4. bias / time-embedding grads ------
@pytest.mark.parametrize("backend,m,n,rpg,ld,copy,accumulate", _backend_params(
    [(512, 320, None, 0, True, True),          # bias gradient + bf16 copy of dy (bias_grad_and_cast)
     (2 * 16, 128, 16, 0, True, False),        # per-sample time-embedding gradient, hw = 16 (TINY)
     (3 * 4, 960, 4, 0, True, False),          # hw = 4
     (2, 320, None, 0, False, True),           # conv1 bias from the per-sample sums: m = batch
     (40, 960, None, 0, False, True),
     (300, 960, None, 1024, True, True)],      # a column slice of a wider gradient (ld > n), m not a multiple of 64
    [(2 * 4096, 320, 4096, 0, True, False), (40 * 64, 1280, 64, 0, True, False), (2 * 4096, 320, None, 0, True, True),
     (40 * 16, 960, 16, 0, True, False), (40 * 1024, 640, 1024, 0, True, False)]))
def test_colsum_cast(backend, m, n, rpg, ld, copy, accumulate):
    be = Backend(backend)
    g = torch.Generator().manual_seed(37 + m + n)
    pitch = ld or n
    dyw = rnd(g, m, pitch)
    groups = m // (rpg or m)
    old = rnd(g, groups, n)
    yb = Guarded(m, n, BF16, be.dev) if copy else None
    out = Guarded(groups, n, F32, be.dev, init=old if accumulate else None)
    be.ops.colsum_cast(dyw.to(be.dev), m, n, y_bf16=yb.view if copy else None, out=out.view, rows_per_group=rpg,
                       accumulate=accumulate, ld=ld)
    be.sync()
    dy = dyw[:, :n].double()
    if copy:
        assert torch.equal(yb.view.cpu(), dyw[:, :n].to(BF16))
        yb.check("colsum_cast bf16 copy")
    check_sum("colsum", out.view.cpu(), dy.reshape(groups, -1, n).sum(1), dy.abs().reshape(groups, -1, n).sum(1),
              old=old if accumulate else None)
    out.check("colsum_cast sums")


@pytest.mark.parametrize("backend,m,n,ld", _backend_params([(300, 2560, 0), (130, 10240, 0), (200, 640, 1024)],
                                                           [(4100, 5120, 0), (2 * 4096, 2560, 0)]))
def test_colsum_bf16(backend, m, n, ld):
    """GEGLU bias gradient (unet.py:693): column sums of the bf16 [M, 8C] gradient, accumulated into the bias grad"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(41 + m)
    x = rnd(g, m, ld or n).to(BF16)
    old = rnd(g, 1, n)
    out = Guarded(1, n, F32, be.dev, init=old)
    be.ops.colsum_bf16(x.to(be.dev), m, n, out.view, accumulate=True, ld=ld)
    be.sync()
    xv = x[:, :n].double()
    check_sum("colsum", out.view.cpu(), xv.sum(0, keepdim=True), xv.abs().sum(0, keepdim=True), old=old)
    out.check("colsum_bf16")


def _silu(v):
    return v * torch.sigmoid(v)


@pytest.mark.parametrize("backend,pattern,batch", _backend_params(
    [(p, b) for p in ("linear_1", "linear_2", "time_emb_proj") for b in (1, 2, 16, 40)]))
def test_dense_small_bwd(backend, pattern, batch):
    """the time-embedding MLP and the resnets' time_emb_proj (unet.py:580-587, 624): te = 1280.
    linear_1: silu_out, no dx.  linear_2: silu_out, dx.  time_emb_proj: no bias, dx accumulated over a chain of calls."""
    be = Backend(backend)
    ops, dev = be.ops, be.dev
    g = torch.Generator().manual_seed(43 + batch)
    te = 1280
    if pattern == "linear_1":
        x = torch.cat([torch.cos(rnd(g, batch, 160)), torch.sin(rnd(g, batch, 160))], 1)   # sincos of a timestep
        layers = [(320, te, True)]
    elif pattern == "linear_2":
        x = _silu(rnd(g, batch, te))
        layers = [(te, te, True)]
    else:
        x = _silu(rnd(g, batch, te))
        layers = [(te, 320, False), (te, 640, False), (te, 1280, False), (te, 320, False)]
    k = x.shape[1]
    want_dx = pattern != "linear_1"
    dx = Guarded(batch, k, F32, dev) if want_dx else None
    dx_ref = torch.zeros(batch, k, dtype=F64)
    dx_terms = torch.zeros(batch, k, dtype=F64)
    for i, (kk, n, silu_out) in enumerate(layers):
        w = rnd(g, kk, n, scale=kk ** -0.5)
        bias = rnd(g, n, scale=0.1) if pattern != "time_emb_proj" else None
        dy = rnd(g, batch, n)
        dw_old, db_old = rnd(g, kk, n, scale=0.1), rnd(g, 1, n, scale=0.1)
        dw = Guarded(kk, n, F32, dev, init=dw_old, extra_rows=1)
        db = Guarded(1, n, F32, dev, init=db_old, extra_rows=1)
        dpre = torch.empty(batch, n, device=dev)
        ops.dense_small_bwd(x.to(dev), w.to(dev), bias.to(dev) if bias is not None else None, dy.to(dev), dpre, dw.view,
                            db.view[0], dx.view if want_dx else None, batch, kk, n, silu_out=silu_out,
                            dx_accumulate=i > 0)
        be.sync()
        # reference: float64 autograd of y = act(x @ w + bias)
        xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
        br = (bias.double() if bias is not None else torch.zeros(n, dtype=F64)).requires_grad_(True)
        pre = xr @ wr + br
        pre.retain_grad()
        (_silu(pre) if silu_out else pre).backward(dy.double())
        # the summed terms of dW, db and dx are built from dpre = dy * silu'(pre).  The kernel recomputes pre as an fp32
        # dot product of K terms, so silu'(pre) carries an absolute error of ~1e-6 even where it is near zero: each term
        # counts at least 0.1 |dy| in the bound
        dpre = pre.grad.abs() + (0.1 * dy.double().abs() if silu_out else 0)
        check_sum(f"dw{i}", dw.view.cpu(), wr.grad, x.double().abs().t() @ dpre, old=dw_old)
        check_sum(f"db{i}", db.view.cpu(), br.grad[None], dpre.sum(0, keepdim=True), old=db_old)
        dw.check("dense_small_bwd dw")
        db.check("dense_small_bwd db")
        dx_ref += xr.grad
        dx_terms += dpre @ w.double().abs().t()
        if want_dx:
            check_sum(f"dx{i}", dx.view.cpu(), dx_ref, dx_terms)
            dx.check("dense_small_bwd dx")


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("backend,rows,cols,lds,ldd", _backend_params(
    [(100, 320, 960, 640), (64, 640, 640, 1280), (7, 128, 192, 128)], [(2 * 4096, 320, 960, 320)]))
def test_copy2d(backend, rows, cols, lds, ldd, accumulate):
    """dst[r, :cols] (+)= src[r, :cols] with different row pitches (unet.py:488-498 put(), 511, 652); the columns past
    ``cols`` and the rows after the last are untouched.  Both modes are exact (one fp32 add)."""
    be = Backend(backend)
    g = torch.Generator().manual_seed(47 + rows)
    src = rnd(g, rows, lds)
    dst = Guarded(rows, ldd, F32, be.dev)        # the whole pitched row is the view: columns >= cols must survive
    before = dst.view.clone().cpu()
    be.ops.copy2d(src.to(be.dev), lds, dst.view, ldd, rows, cols, accumulate=accumulate)
    be.sync()
    got = dst.view.cpu()
    want = before.clone()
    want[:, :cols] = before[:, :cols] + src[:, :cols] if accumulate else src[:, :cols]
    assert torch.equal(got, want)
    dst.check("copy2d")


# ----------------------------------------------------------------------------------- 2. attention backward ------
def _attention_ref(q, k, v, do):
    """float64 (dq, dk, dv) of O = softmax(Q K^T / 8) V for one (sample, head): [n, 64] operands"""
    q, k, v = (t.double().requires_grad_(True) for t in (q, k, v))
    o = torch.softmax(q @ k.t() * 0.125, -1) @ v
    o.backward(do.double())
    return q.grad, k.grad, v.grad


class _ErrAcc:
    """max-abs and L2 errors of a gradient assembled one (sample, head) block at a time"""

    def __init__(self):
        self.max_err = self.max_ref = self.sq_err = self.sq_ref = 0.0

    def add(self, got, ref):
        d = got.double() - ref
        self.max_err = max(self.max_err, d.abs().max().item())
        self.max_ref = max(self.max_ref, ref.abs().max().item())
        self.sq_err += (d * d).sum().item()
        self.sq_ref += (ref * ref).sum().item()

    def check(self, name):
        e_max, e_l2 = self.max_err / self.max_ref, (self.sq_err / self.sq_ref) ** 0.5
        _record(name, max=e_max, l2=e_l2)
        assert e_max <= ATT_MAX and e_l2 <= ATT_L2, \
            f"{name}: max err {e_max:.3g} * max|ref| (bound {ATT_MAX}), relative L2 {e_l2:.3g} (bound {ATT_L2})"


def _check_delta(delta, out, do, b, heads, n):
    """delta[b, h, q] = sum_d dO * O over the head's 64 columns (out and dO as the kernel read them)"""
    prod = (out.double() * do.double()).reshape(b, n, heads, 64)
    check_sum("delta", delta.reshape(b, heads, n).permute(0, 2, 1), prod.sum(-1), prod.abs().sum(-1))


@pytest.mark.gpu
@pytest.mark.parametrize("b,heads,n", [(2, 5, 4096), (2, 10, 1024), (2, 20, 256), (2, 20, 64), (2, 2, 16), (2, 2, 4),
                                       (2, 2, 300)])
def test_self_attention_bwd_fused_qkv(b, heads, n):
    """self-attention backward as unet.py:728: q/k/v are column slices of ONE [b*n, 3C] buffer and dq/dk/dv of one
    [b*n, 3C] gradient buffer (here with the pitch widened by a 64-column sentinel block).  The reference is built one
    (sample, head) at a time so that the 4096-token case stays under 1 GB of float64."""
    from ddpo_b200 import ops
    dev = "cuda"
    c = heads * 64
    m = b * n
    ld = 3 * c + 64
    g = torch.Generator().manual_seed(53 + n + heads)
    qkv = rnd(g, m, ld).to(BF16).to(dev)
    do = rnd(g, m, c).to(BF16).to(dev)
    out = torch.empty(m, c, dtype=BF16, device=dev)
    lse = torch.empty(b, heads, n, device=dev)
    ops.attention_fwd(qkv, qkv[:, c:], qkv[:, 2 * c:], out, b, heads, n, n, ld, ld, ld, c, lse=lse)

    def run(bb, r0):
        dq = Guarded(bb * n, 3 * c, BF16, dev, extra_cols=64)
        delta = Guarded(bb * heads, n, F32, dev)
        rows = slice(r0 * n, (r0 + bb) * n)
        qs = qkv[rows]
        ops.attention_bwd(qs, qs[:, c:], qs[:, 2 * c:], out[rows], do[rows], lse[r0:r0 + bb], delta.view, dq.buf,
                          dq.buf[:, c:], dq.buf[:, 2 * c:], bb, heads, n, n, ld, ld, ld, c, c, ld, ld, ld)
        torch.cuda.synchronize()
        dq.check("dqkv")
        delta.check("delta")
        return dq.view, delta.view

    dqkv, delta = run(b, 0)
    _check_delta(delta, out, do, b, heads, n)
    acc = [_ErrAcc() for _ in range(3)]
    for s in range(b):
        rows = slice(s * n, (s + 1) * n)
        for h in range(heads):
            cols = [slice(i * c + h * 64, i * c + (h + 1) * 64) for i in range(3)]
            refs = _attention_ref(qkv[rows, cols[0]], qkv[rows, cols[1]], qkv[rows, cols[2]], do[rows, h * 64:(h + 1) * 64])
            for i in range(3):
                acc[i].add(dqkv[rows, cols[i]], refs[i])
    for i, name in enumerate(("dq", "dk", "dv")):
        acc[i].check(name)
    # deterministic, no atomics: a second run and the last sample computed alone give the same bits
    dqkv2, delta2 = run(b, 0)
    assert torch.equal(dqkv, dqkv2) and torch.equal(delta, delta2)
    alone, _ = run(1, b - 1)
    assert torch.equal(alone, dqkv[(b - 1) * n:])


@pytest.mark.gpu
@pytest.mark.parametrize("b,heads,n", [(2, 2, 16), (2, 2, 4), (2, 5, 64)])
def test_cross_attention_bwd(b, heads, n):
    """cross-attention backward as unet.py:711: q pitch C, k/v column slices of the [b*77, 2C] context projection, dq
    [b*n, C], dk/dv column slices of one [b*77, 2C] buffer; n = 16 and 4 are TINY's two lowest levels"""
    from ddpo_b200 import ops
    dev = "cuda"
    c, L = heads * 64, 77
    m = b * n
    g = torch.Generator().manual_seed(59 + n)
    q = rnd(g, m, c).to(BF16).to(dev)
    kv = rnd(g, b * L, 2 * c).to(BF16).to(dev)
    do = rnd(g, m, c).to(BF16).to(dev)
    out = torch.empty(m, c, dtype=BF16, device=dev)
    lse = torch.empty(b, heads, n, device=dev)
    ops.attention_fwd(q, kv, kv[:, c:], out, b, heads, n, L, c, 2 * c, 2 * c, c, lse=lse)

    def run(bb, s0):
        dq = Guarded(bb * n, c, BF16, dev)
        dkv = Guarded(bb * L, 2 * c, BF16, dev)
        delta = Guarded(bb * heads, n, F32, dev)
        qr, kr = slice(s0 * n, (s0 + bb) * n), slice(s0 * L, (s0 + bb) * L)
        ops.attention_bwd(q[qr], kv[kr], kv[kr, c:], out[qr], do[qr], lse[s0:s0 + bb], delta.view, dq.view, dkv.view,
                          dkv.view[:, c:], bb, heads, n, L, c, 2 * c, 2 * c, c, c, c, 2 * c, 2 * c)
        torch.cuda.synchronize()
        for t, nm in ((dq, "dq"), (dkv, "dkv"), (delta, "delta")):
            t.check(nm)
        return dq.view, dkv.view, delta.view

    dq, dkv, delta = run(b, 0)
    _check_delta(delta, out, do, b, heads, n)
    acc = [_ErrAcc() for _ in range(3)]
    for s in range(b):
        qr, kr = slice(s * n, (s + 1) * n), slice(s * L, (s + 1) * L)
        for h in range(heads):
            hc = slice(h * 64, (h + 1) * 64)
            refs = _attention_ref(q[qr, hc], kv[kr, hc], kv[kr, c + h * 64:c + (h + 1) * 64], do[qr, hc])
            acc[0].add(dq[qr, hc], refs[0])
            acc[1].add(dkv[kr, hc], refs[1])
            acc[2].add(dkv[kr, c + h * 64:c + (h + 1) * 64], refs[2])
    for i, name in enumerate(("dq", "dk", "dv")):
        acc[i].check(name)
    again = run(b, 0)
    assert all(torch.equal(x, y) for x, y in zip((dq, dkv, delta), again))
    alone = run(1, b - 1)
    assert torch.equal(alone[0], dq[(b - 1) * n:]) and torch.equal(alone[1], dkv[(b - 1) * L:])


# ---------------------------------------------------------------------------------- 3. GroupNorm backward ------
def _gn_case(b, h, w, c0, c1, seed):
    g = torch.Generator().manual_seed(seed)
    hw, c = h * w, c0 + c1
    return dict(x0=rnd(g, b * hw, c0, scale=2.0, shift=0.5), x1=rnd(g, b * hw, c1) if c1 else None,
                sc=rnd(g, c, scale=0.1, shift=1.0), bi=rnd(g, c, scale=0.1), dy=rnd(g, b * hw, c).to(BF16),
                old=rnd(g, b * hw, c, scale=0.5), dsc_old=rnd(g, c), dbi_old=rnd(g, c))


def _gn_run(case, b, hw, c0, c1):
    """norm1 backward of a resnet as unet.py:636-659: forward first (it leaves mean / rstd in the workspace), then the
    backward accumulating into the gradient the shortcut dgrad (two sources: ``dcat``, x1's part a column slice of it,
    both with pitch cin) or the skip connection (one source) already wrote"""
    from ddpo_b200 import ops
    dev = "cuda"
    c = c0 + c1
    x0, x1 = case["x0"].to(dev), case["x1"].to(dev) if c1 else None
    sc, bi = case["sc"].to(dev), case["bi"].to(dev)
    ws = torch.zeros(ops.groupnorm_workspace_floats(b, hw, c), device=dev)
    a = torch.empty(b * hw, c, dtype=BF16, device=dev)
    ops.groupnorm_fwd(x0, sc, bi, ws, b, hw, c0, x1=x1, c1=c1, silu=True, y_bf16=a)
    dcat = Guarded(b * hw, c, F32, dev, init=case["old"])
    dsc = Guarded(1, c, F32, dev, init=case["dsc_old"])
    dbi = Guarded(1, c, F32, dev, init=case["dbi_old"])
    ops.groupnorm_bwd(x0, sc, bi, ws, b, hw, c0, case["dy"].to(dev), dcat.view, dsc.view, dbi.view, x1=x1, c1=c1,
                      dx1=dcat.view[:, c0:] if c1 else None, silu=True, accumulate=True, ldd0=c if c1 else 0,
                      ldd1=c if c1 else 0)
    torch.cuda.synchronize()
    for t, nm in ((dcat, "dx"), (dsc, "dscale"), (dbi, "dbias")):
        t.check(nm)
    return dcat.view, dsc.view[0], dbi.view[0]


GN_CASES = [(4, 8, 8, 1280, 1280), (4, 16, 16, 1280, 640), (4, 32, 32, 640, 320), (4, 64, 64, 320, 320),
            (4, 64, 64, 640, 320), (2, 16, 32, 640, 320), (40, 64, 64, 320, 0), (40, 32, 32, 640, 320)]


@pytest.mark.gpu
@pytest.mark.parametrize("b,h,w,c0,c1", GN_CASES)
def test_groupnorm_bwd_resnet_norm1(b, h, w, c0, c1):
    hw, c = h * w, c0 + c1
    case = _gn_case(b, h, w, c0, c1, 61 + c + hw + b)
    dx, dsc, dbi = _gn_run(case, b, hw, c0, c1)
    dev = "cuda"
    x = case["x0"] if not c1 else torch.cat([case["x0"], case["x1"]], 1)
    xr = x.double().to(dev).requires_grad_(True)
    scr, bir = case["sc"].double().to(dev).requires_grad_(True), case["bi"].double().to(dev).requires_grad_(True)
    y = F.group_norm(xr.reshape(b, hw, c).permute(0, 2, 1), 32, scr, bir, 1e-5)
    dyd = case["dy"].double().to(dev).reshape(b, hw, c).permute(0, 2, 1)
    F.silu(y).backward(dyd)
    check_close("dx", dx.double() - case["old"].double().to(dev), xr.grad, F32_MAX, F32_L2)
    # dscale / dbias: sums over (sample, pixel) of dy' * xhat and dy', dy' = dy * silu'(y)
    with torch.no_grad():
        yd = y.detach()
        s = torch.sigmoid(yd)
        dyp = dyd * s * (1 + yd * (1 - s))
        xhat = (yd - bir[None, :, None]) / scr[None, :, None]
    check_sum("dscale", dsc, scr.grad, (dyp * xhat).abs().sum(dim=(0, 2)), tol=2 * SUM_TOL, old=case["dsc_old"].to(dev))
    check_sum("dbias", dbi, bir.grad, dyp.abs().sum(dim=(0, 2)), tol=2 * SUM_TOL, old=case["dbi_old"].to(dev))

