"""The parameter side of the U-Net backward pass (ddpo_b200/unet.py, ``UNet.backward``) layer by layer: every kernel
that writes into the flat fp32 gradient buffer ``UNet.grads``, called with the arguments unet.py passes, and the two
optimizer kernels that consume that buffer.  test_backward_layers.py covers the data-gradient side.

Conventions (the harness is tests/_layer_check.py):
- the reference is float64, computed from the same bf16- or fp32-rounded operands the kernel reads; large references
  run on the test's device (one ``X_shifted^T @ dY`` per tap, not a CPU convolution);
- every parameter gradient lands in a ``FlatSlot``: a view at a 64-float aligned offset of a 1-D fp32 buffer, as
  ``UNet.g(name)`` slices ``UNet.grads``.  The slot starts from a non-zero prior gradient, because the train pass always
  accumulates, and the neighbouring parameters must come back bit-identical;
- reductions are bounded per element by ``SUM_TOL * sum|terms|`` plus one fp32 rounding of the accumulate-into
  (``check_sum``); elementwise outputs get max-abs and relative-L2 bounds (``check_close``); the optimizer's bounds are
  derived below from the kernel's rounding steps.

Small cases also run on the torch-CPU emulation of the ops (tests/_cpu_ops_emulator.py); CUDA cases carry the ``gpu``
mark.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from _layer_check import (BF16, F32, F32_L2, F32_MAX, SUM_TOL, Backend, FlatSlot, Guarded, _backend_params,
                          _current_node, _record, check_close, check_sum, rnd)  # noqa: F401

U32 = 2.0 ** -24                      # unit roundoff of fp32 (round to nearest)
U_BF16 = 2.0 ** -8                    # unit roundoff of bf16


def _rows(t_nchw):
    """NCHW -> [b*h*w, c]"""
    return t_nchw.permute(0, 2, 3, 1).reshape(-1, t_nchw.shape[1])


# --------------------------------------------------------------------------------------------------- 1. wgrad ------
def _wgrad_ref(x, dy, conv, taps=1, stride=1):
    """float64 dW[(tap, c_in), n] = sum over output pixels of X[the input pixel the tap reads] * dY, and the same sum
    over |X| |dY|.  x: [rows, c_in] (NHWC rows of the input, size (b, h*stride, w*stride)), dy: [pixels, n]."""
    xd, dyd = x.double(), dy.double()
    if conv is None:
        return xd.t() @ dyd, xd.abs().t() @ dyd.abs()
    b, h, w = conv
    x4 = xd.reshape(b, h * stride, w * stride, -1)
    if taps == 9:
        x4 = F.pad(x4, (0, 0, 1, 1, 1, 1))
    refs, terms = [], []
    for tap in range(taps):
        ky, kx = divmod(tap, 3) if taps == 9 else (0, 0)
        xs = x4[:, ky:ky + stride * h:stride, kx:kx + stride * w:stride].reshape(b * h * w, -1)
        refs.append(xs.t() @ dyd)
        terms.append(xs.abs().t() @ dyd.abs())
    return torch.cat(refs), torch.cat(terms)


def _wgrad_splits(conv, m, cin, n, taps, stride=1):
    """how many pixel splits the library's planner picks (1: the GEMM epilogue adds into dW; > 1: partials in the
    workspace, summed by wgrad_reduce_kernel) and the workspace floats it asks for"""
    from ddpo_b200._lib import WgradArgs, lib
    a = WgradArgs()
    if conv is not None:
        a.is_conv, a.batch, a.h, a.w, a.m = 1, conv[0], conv[1], conv[2], 0
    else:
        a.is_conv, a.m = 0, m
    a.c0, a.c1, a.n, a.taps, a.conv_stride = cin, 0, n, taps, stride
    need = int(lib().ddpo_wgrad_workspace_floats(ctypes.byref(a)))
    return (need // (taps * cin * n) if need else 1), need


class _OwnWorkspace:
    """Hands ``ops.wgrad`` a workspace the test owns: exactly the floats the planner asks for, at ``offset`` floats
    into a buffer whose remaining floats are seeded noise that must come back unchanged.  A kernel that writes past
    the workspace it asked for then lands in memory the test checks, not in someone else's allocation."""

    def __init__(self, ops, dev, need, offset=0, tail=1 << 20):
        self.ops, self.key = ops, torch.empty(0, device=dev).device
        g = torch.Generator().manual_seed(97)
        self.buf = torch.randn(offset + need + tail, generator=g).to(dev)
        self.snapshot_tail = self.buf[offset + need:].clone()
        self.view = self.buf[offset:offset + need]
        self.need = need

    def __enter__(self):
        self.saved = self.ops._WGRAD_WS.get(self.key)
        if self.need:
            self.ops._WGRAD_WS[self.key] = self.view
        return self

    def __exit__(self, *exc):
        if self.saved is None:
            self.ops._WGRAD_WS.pop(self.key, None)
        else:
            self.ops._WGRAD_WS[self.key] = self.saved

    def check(self, what):
        assert torch.equal(self.buf[-self.snapshot_tail.numel():], self.snapshot_tail), f"{what}: write past the workspace"


def _wgrad_into_slots(be, calls, slots, plan):
    """run the wgrad ``calls`` (kwargs for ops.wgrad without dw) into their slots; on CUDA with a test-owned
    workspace sized for ``plan`` = (conv, m, c_in, n, taps, stride).  Returns the planner's split count."""
    splits, need = 1, 0
    if not be.emulated:
        splits, need = _wgrad_splits(*plan)
    ws = _OwnWorkspace(be.ops, be.dev, need) if not be.emulated else None
    if ws is not None:
        with ws:
            for kw, slot in zip(calls, slots):
                be.ops.wgrad(dw=slot.view, **kw)
            be.sync()
        ws.check("wgrad")
    else:
        for kw, slot in zip(calls, slots):
            be.ops.wgrad(dw=slot.view, **kw)
    return splits


def _ghost_rows(n):
    """floats of neighbouring parameters after a wgrad slot: 128 rows of dW, the most a 128-channel block of the
    kernel could overhang the last input channel, so that a missing channel guard writes into memory the test checks"""
    return 128 * n


# (site, b, h, w, c_in, n): h, w are the spatial size of the site's input (x0); linear sites have m = b * h * w rows
WGRAD_SMALL = [("conv2", 2, 8, 8, 64, 64), ("conv1", 1, 4, 8, 192, 128), ("shortcut", 2, 4, 4, 192, 64),
               ("down", 2, 8, 8, 64, 64), ("up", 1, 4, 4, 128, 64), ("linear", 2, 4, 4, 64, 512)]
WGRAD_LARGE = [
    # resnet conv2 (3x3, x0 = a2)
    ("conv2", 2, 64, 64, 320, 320), ("conv2", 2, 32, 32, 640, 640), ("conv2", 2, 16, 16, 1280, 1280),
    ("conv2", 2, 8, 8, 1280, 1280), ("conv2", 40, 64, 64, 320, 320),
    # resnet conv1 (3x3, x0 = a) at the up-block widths; at 960 the last 128-channel block is half empty
    ("conv1", 2, 8, 8, 2560, 1280), ("conv1", 2, 16, 16, 1920, 1280), ("conv1", 2, 32, 32, 960, 640),
    ("conv1", 2, 64, 64, 640, 320),
    # conv_shortcut (taps = 1, conv mode, x0 = raw)
    ("shortcut", 2, 8, 8, 2560, 1280), ("shortcut", 2, 32, 32, 960, 640),
    # downsampler (stride 2; h, w of the input)
    ("down", 2, 64, 64, 320, 320), ("down", 2, 32, 32, 640, 640), ("down", 2, 16, 16, 1280, 1280),
    # upsampler conv over the 2x input (h, w before the upsample)
    ("up", 2, 8, 8, 1280, 1280), ("up", 2, 16, 16, 1280, 1280), ("up", 2, 32, 32, 640, 640),
    # proj_in / proj_out / to_out_0 / attn2 to_q (C -> C)
    ("linear", 2, 64, 64, 320, 320), ("linear", 2, 32, 32, 640, 640), ("linear", 2, 16, 16, 1280, 1280),
    ("linear", 2, 8, 8, 1280, 1280), ("linear", 40, 32, 32, 640, 640),
    # GEGLU ff/net_0/proj (N = 8C) and ff/net_2 (K = 4C)
    ("linear", 2, 8, 8, 1280, 10240), ("linear", 2, 32, 32, 640, 5120), ("linear", 2, 8, 8, 5120, 1280),
    ("linear", 2, 64, 64, 1280, 320),
    # TINY / SMALL widths: N = 64 or 128 takes only the remainder launch
    ("conv2", 2, 32, 32, 64, 64), ("conv1", 2, 32, 32, 192, 64), ("linear", 2, 16, 16, 128, 128),
    ("linear", 2, 32, 32, 64, 512), ("linear", 2, 32, 32, 256, 64)]


def _site_args(site, b, h, w, cin):
    """(conv, m, taps, stride, x rows, dy rows) of a wgrad call site"""
    if site in ("conv2", "conv1"):
        return (b, h, w), None, 9, 1, b * h * w, b * h * w
    if site == "shortcut":
        return (b, h, w), None, 1, 1, b * h * w, b * h * w
    if site == "down":
        return (b, h // 2, w // 2), None, 9, 2, b * h * w, b * h * w // 4
    if site == "up":
        return (b, 2 * h, 2 * w), None, 9, 1, 4 * b * h * w, 4 * b * h * w
    return None, b * h * w, 1, 1, b * h * w, b * h * w


@pytest.mark.parametrize("backend,site,b,h,w,cin,n", _backend_params(WGRAD_SMALL, WGRAD_LARGE))
def test_wgrad_call_sites(backend, site, b, h, w, cin, n):
    """dW (+)= X^T dY at each unet.py call site (unet.py:533, 549, 605, 629, 634, 677, 686, 694, 703, 713, 723, 739),
    into a flat-buffer slot with a non-zero prior; a second run from the same prior gives the same bits"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(101 + b + h + cin + n)
    conv, m, taps, stride, xr, dr = _site_args(site, b, h, w, cin)
    if site == "up":     # the upsampler conv reads nearest-2x copies of its input
        x = rnd(g, b, h, w, cin).repeat_interleave(2, 1).repeat_interleave(2, 2).reshape(xr, cin)
    else:
        x = rnd(g, xr, cin)
    x = x.to(BF16).to(be.dev)
    dy = rnd(g, dr, n).to(BF16).to(be.dev)
    prior = rnd(g, taps * cin, n, scale=float(dr) ** 0.5)     # of the order of one accumulated gradient
    kw = dict(dy=dy, n=n, x0=x, c0=cin, conv=conv, m=m, taps=taps, stride=stride)
    plan = (conv, m, cin, n, taps, stride)
    slots = [FlatSlot(taps * cin, n, be.dev, prior, after=_ghost_rows(n)) for _ in range(2 if not be.emulated else 1)]
    splits = _wgrad_into_slots(be, [kw] * len(slots), slots, plan)
    _record("plan", splits=splits)
    ref, terms = _wgrad_ref(x, dy, conv, taps, stride)
    # with splits > 1 the prior is the first of 1 + splits fp32 adds; its share of the rounding error,
    # splits * 2^-24 * |prior|, is far below SUM_TOL * sum|terms| at these magnitudes
    check_sum("dw", slots[0].view, ref, terms, old=slots[0].prior())
    for s in slots:
        s.check("wgrad")
    if len(slots) > 1:
        assert torch.equal(slots[0].view, slots[1].view), "two runs from the same prior differ"


@pytest.mark.gpu
def test_wgrad_call_sites_cover_both_planner_paths():
    """the cases above exercise both the in-epilogue accumulate (splits == 1) and the split reduction (splits > 1)"""
    seen = set()
    for site, b, h, w, cin, n in WGRAD_LARGE:
        conv, m, taps, stride, _, _ = _site_args(site, b, h, w, cin)
        seen.add(_wgrad_splits(conv, m, cin, n, taps, stride)[0] > 1)
    assert seen == {False, True}


@pytest.mark.parametrize("backend,b,hw,c", _backend_params([(2, 16, 64)], [(2, 4096, 320), (2, 1024, 640), (2, 64, 1280),
                                                                         (40, 1024, 640)]))
def test_wgrad_self_attention_qkv_slices(backend, b, hw, c):
    """attn1 to_q / to_k / to_v (unet.py:730): dY is the column slice dqkv[:, i*C:] of ONE [b*hw, 3C] gradient, pitch 3C;
    the three results are the three column blocks of one reference"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(103 + hw + c)
    m = b * hw
    ln1 = rnd(g, m, c).to(BF16).to(be.dev)
    dqkv = rnd(g, m, 3 * c).to(BF16).to(be.dev)
    slots = [FlatSlot(c, c, be.dev, rnd(g, c, c, scale=m ** 0.5), after=_ghost_rows(c), seed=90 + i) for i in range(3)]
    calls = [dict(dy=dqkv[:, i * c:], ldy=3 * c, n=c, x0=ln1, c0=c, m=m) for i in range(3)]
    splits = _wgrad_into_slots(be, calls, slots, (None, m, c, c, 1, 1))
    _record("plan", splits=splits)
    ref, terms = _wgrad_ref(ln1, dqkv, None)
    for i, nm in enumerate(("to_q", "to_k", "to_v")):
        cols = slice(i * c, (i + 1) * c)
        check_sum(nm, slots[i].view, ref[:, cols], terms[:, cols], old=slots[i].prior())
        slots[i].check(nm)


@pytest.mark.parametrize("backend,b,c,dctx", _backend_params([(2, 64, 64)], [(2, 320, 1024), (2, 640, 1024), (2, 1280, 1024),
                                                                           (2, 320, 768), (2, 1280, 768), (2, 128, 64),
                                                                           (40, 640, 1024)]))
def test_wgrad_cross_attention_kv_slices(backend, b, c, dctx):
    """attn2 to_k / to_v (unet.py:714-715): X is the bf16 text context (m = b*77 rows, so the last 64-row block is
    ragged), dY the column slices dkv[:, :C] and dkv[:, C:] of one [b*77, 2C] gradient, pitch 2C.  dctx = 1024 (SD2),
    768 (SD1), 64 (TINY)."""
    be = Backend(backend)
    g = torch.Generator().manual_seed(107 + c + dctx + b)
    m = b * 77
    ctx = rnd(g, m, dctx).to(BF16).to(be.dev)
    dkv = rnd(g, m, 2 * c).to(BF16).to(be.dev)
    slots = [FlatSlot(dctx, c, be.dev, rnd(g, dctx, c, scale=m ** 0.5), after=_ghost_rows(c), seed=80 + i)
             for i in range(2)]
    calls = [dict(dy=dkv[:, i * c:], ldy=2 * c, n=c, x0=ctx, c0=dctx, m=m) for i in range(2)]
    splits = _wgrad_into_slots(be, calls, slots, (None, m, dctx, c, 1, 1))
    _record("plan", splits=splits)
    ref, terms = _wgrad_ref(ctx, dkv, None)
    for i, nm in enumerate(("to_k", "to_v")):
        cols = slice(i * c, (i + 1) * c)
        check_sum(nm, slots[i].view, ref[:, cols], terms[:, cols], old=slots[i].prior())
        slots[i].check(nm)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["dw", "workspace"])
def test_wgrad_rejects_misaligned_buffers(which):
    """dw and the workspace must be 16-byte aligned: the split reduction reads and writes them as float4.  A buffer 8
    bytes off is refused on the host, before anything is launched, and no buffer changes."""
    from ddpo_b200 import ops
    from ddpo_b200._lib import DdpoError
    dev = "cuda"
    m, c = 8192, 320
    splits, need = _wgrad_splits(None, m, c, c, 1)
    assert splits > 1, "the shape must take the split reduction"
    g = torch.Generator().manual_seed(109)
    x = rnd(g, m, c).to(BF16).to(dev)
    dy = rnd(g, m, c).to(BF16).to(dev)
    dw_buf = rnd(g, c * c + 64).to(dev)
    dw = dw_buf[2:2 + c * c].view(c, c) if which == "dw" else dw_buf[:c * c].view(c, c)
    before = dw_buf.clone()
    with _OwnWorkspace(ops, dev, need, offset=2 if which == "workspace" else 0) as ws:
        ws_before = ws.buf.clone()
        with pytest.raises(DdpoError, match="16-byte aligned"):
            ops.wgrad(dy=dy, n=c, x0=x, c0=c, m=m, dw=dw)
        torch.cuda.synchronize()
        assert torch.equal(ws.buf, ws_before)
    assert torch.equal(dw_buf, before)


# ------------------------------------------------------------------------------------ 2. norm parameter grads ------
@pytest.mark.parametrize("backend,m,c", _backend_params([(100, 64), (300, 128)],
                                                        [(2 * 4096, 320), (2 * 1024, 640), (2 * 256, 1280), (2 * 16, 64),
                                                         (4100, 1280), (40 * 4096, 320), (40 * 1024, 640)]))
def test_layernorm_bwd_transformer_chain(backend, m, c):
    """the three LayerNorm backwards of one transformer block as _transformer_bwd makes them (unet.py:698-734): norm3,
    norm2, norm1 in turn, sharing one workspace, each adding its input gradient into the same fp32 d_h from a bf16 dy,
    and its dscale / dbias into flat-buffer slots"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(113 + m + c)
    ws = torch.zeros(be.ops.layernorm_bwd_workspace_floats(m, c), device=be.dev)
    d_h = Guarded(m, c, F32, be.dev, init=rnd(g, m, c, scale=0.5))
    for nm in ("norm3", "norm2", "norm1"):
        x = rnd(g, m, c, scale=2.0, shift=0.5)
        sc, bi = rnd(g, c, scale=0.1, shift=1.0), rnd(g, c, scale=0.1)
        dy = rnd(g, m, c).to(BF16)
        dsc = FlatSlot(1, c, be.dev, rnd(g, c, scale=10.0), seed=70)
        dbi = FlatSlot(1, c, be.dev, rnd(g, c, scale=10.0), seed=71)
        xd, scd, bid = x.to(be.dev), sc.to(be.dev), bi.to(be.dev)
        st = torch.zeros(m, 2, device=be.dev)
        be.ops.layernorm_fwd(xd, scd, bid, torch.empty(m, c, dtype=BF16, device=be.dev), m, c, stats=st)
        old = d_h.view.clone()
        be.ops.layernorm_bwd(xd, scd, st, dy.to(be.dev), d_h.view, dsc.view[0], dbi.view[0], ws, m, c, accumulate=True)
        be.sync()
        xr = xd.double().requires_grad_(True)
        scr, bir = scd.double().requires_grad_(True), bid.double().requires_grad_(True)
        y = F.layer_norm(xr, (c,), scr, bir, 1e-5)
        dyd = dy.double().to(be.dev)
        y.backward(dyd)
        xhat = (y.detach() - bir.detach()) / scr.detach()
        check_close(f"{nm} dx", d_h.view.double() - old.double(), xr.grad, F32_MAX, F32_L2)
        # the statistics come from the fp32 forward pass, as in the GroupNorm checks: 2 * SUM_TOL
        check_sum(f"{nm} dscale", dsc.view[0], scr.grad, (dyd * xhat).abs().sum(0), tol=2 * SUM_TOL, old=dsc.prior()[0])
        check_sum(f"{nm} dbias", dbi.view[0], bir.grad, dyd.abs().sum(0), tol=2 * SUM_TOL, old=dbi.prior()[0])
        d_h.check(f"{nm} d_h")
        dsc.check(f"{nm} dscale")
        dbi.check(f"{nm} dbias")


@pytest.mark.parametrize("backend,pattern,b,h,w,c", _backend_params(
    [("transformer_norm", 2, 4, 8, 64), ("conv_norm_out", 2, 4, 8, 64)],
    [("transformer_norm", 2, 64, 64, 320), ("transformer_norm", 2, 32, 32, 640), ("transformer_norm", 2, 16, 16, 1280),
     ("transformer_norm", 2, 8, 8, 1280), ("transformer_norm", 40, 64, 64, 320), ("conv_norm_out", 2, 64, 64, 320),
     ("conv_norm_out", 40, 64, 64, 320), ("conv_norm_out", 2, 32, 32, 64)]))
def test_groupnorm_bwd_param_grads(backend, pattern, b, h, w, c):
    """GroupNorm backward in the two call patterns besides resnet norm1: the transformer ``norm`` (unet.py:743; no
    SiLU, bf16 dy, accumulating into the gradient the residual already has) and ``conv_norm_out`` (unet.py:523; SiLU,
    fp32 dy from conv_out_bwd, a fresh dx).  dscale / dbias accumulate into flat-buffer slots."""
    be = Backend(backend)
    g = torch.Generator().manual_seed(127 + b + h + c)
    hw, m = h * w, b * h * w
    silu = pattern == "conv_norm_out"
    x = rnd(g, m, c, scale=2.0, shift=0.5)
    sc, bi = rnd(g, c, scale=0.1, shift=1.0), rnd(g, c, scale=0.1)
    dy = rnd(g, m, c)
    if not silu:
        dy = dy.to(BF16)
    old = rnd(g, m, c, scale=0.5)
    xd, scd, bid = x.to(be.dev), sc.to(be.dev), bi.to(be.dev)
    ws = torch.zeros(be.ops.groupnorm_workspace_floats(b, hw, c), device=be.dev)
    be.ops.groupnorm_fwd(xd, scd, bid, ws, b, hw, c, silu=silu, y_bf16=torch.empty(m, c, dtype=BF16, device=be.dev))
    dx = Guarded(m, c, F32, be.dev, init=None if silu else old)
    dsc = FlatSlot(1, c, be.dev, rnd(g, c, scale=10.0), seed=72)
    dbi = FlatSlot(1, c, be.dev, rnd(g, c, scale=10.0), seed=73)
    be.ops.groupnorm_bwd(xd, scd, bid, ws, b, hw, c, dy.to(be.dev), dx.view, dsc.view[0], dbi.view[0], silu=silu,
                         accumulate=not silu)
    be.sync()
    xr = xd.double().requires_grad_(True)
    scr, bir = scd.double().requires_grad_(True), bid.double().requires_grad_(True)
    y = F.group_norm(xr.reshape(b, hw, c).permute(0, 2, 1), 32, scr, bir, 1e-5)
    dyd = dy.double().to(be.dev).reshape(b, hw, c).permute(0, 2, 1)
    (F.silu(y) if silu else y).backward(dyd)
    got = dx.view.double() - (0 if silu else old.double().to(be.dev))
    check_close("dx", got, xr.grad, F32_MAX, F32_L2)
    with torch.no_grad():
        yd = y.detach()
        if silu:
            s = torch.sigmoid(yd)
            dyd = dyd * s * (1 + yd * (1 - s))
        xhat = (yd - bir[None, :, None]) / scr[None, :, None]
    check_sum("dscale", dsc.view[0], scr.grad, (dyd * xhat).abs().sum(dim=(0, 2)), tol=2 * SUM_TOL, old=dsc.prior()[0])
    check_sum("dbias", dbi.view[0], bir.grad, dyd.abs().sum(dim=(0, 2)), tol=2 * SUM_TOL, old=dbi.prior()[0])
    dx.check("dx")
    dsc.check("dscale")
    dbi.check("dbias")


# ------------------------------------------------------------------------------------------ 3. stem gradients ------
@pytest.mark.parametrize("backend,b,h,w,c", _backend_params([(2, 8, 8, 64), (1, 4, 8, 32)], [(2, 64, 64, 320), (40, 64, 64, 320)]))
def test_conv_out_bwd_train_pass(backend, b, h, w, c):
    """conv_out backward (unet.py:520): d_yf = conv dgrad of d_eps (fresh), dW and dbias added into flat-buffer slots;
    at 40 x 64^2 pixels the weight gradient goes through the 256-way split reduction.  Two runs from the same prior give
    the same bits."""
    be = Backend(backend)
    g = torch.Generator().manual_seed(131 + b + c)
    m = b * h * w
    x = rnd(g, m, c).to(be.dev)                               # yf, NHWC fp32
    wt = rnd(g, 3, 3, c, 4, scale=(9 * c) ** -0.5).to(be.dev)    # HWIO
    dy = rnd(g, b, 4, h, w).to(be.dev)                         # d_eps, NCHW fp32
    dw_prior, db_prior = rnd(g, 9 * c, 4, scale=m ** 0.5), rnd(g, 1, 4, scale=m ** 0.5)
    runs = []
    for _ in range(1 if be.emulated else 2):
        dx = Guarded(m, c, F32, be.dev)
        dw = FlatSlot(9 * c, 4, be.dev, dw_prior)
        db = FlatSlot(1, 4, be.dev, db_prior, after=64)
        be.ops.conv_out_bwd(x, wt, dy, dx.view, dw.view.view(3, 3, c, 4), db.view[0], b, h, w, c)
        be.sync()
        for t, nm in ((dx, "dx"), (dw, "dw"), (db, "dbias")):
            t.check(nm)
        runs.append((dx.view, dw.view, db.view))
    dyd = dy.double()
    wo = wt.double().permute(3, 2, 0, 1)
    ref_dx = torch.nn.grad.conv2d_input((b, c, h, w), wo, dyd, padding=1)
    terms_dx = torch.nn.grad.conv2d_input((b, c, h, w), wo.abs(), dyd.abs(), padding=1)
    check_sum("dx", runs[0][0], _rows(ref_dx), _rows(terms_dx))
    ref, terms = _wgrad_ref(x, _rows(dy), (b, h, w), 9)
    check_sum("dw", runs[0][1], ref, terms, old=dw_prior.to(be.dev))
    check_sum("dbias", runs[0][2], dyd.sum(dim=(0, 2, 3))[None], dyd.abs().sum(dim=(0, 2, 3))[None],
              old=db_prior.to(be.dev))
    if len(runs) > 1:
        assert all(torch.equal(p, q) for p, q in zip(runs[0], runs[1])), "two runs from the same prior differ"


@pytest.mark.parametrize("backend,b,h,w,c", _backend_params([(2, 8, 8, 64), (1, 4, 8, 96)], [(2, 64, 64, 320), (40, 64, 64, 320)]))
def test_conv_in_wgrad_train_pass(backend, b, h, w, c):
    """conv_in weight gradient (unet.py:573): dW[tap, c_in, c_out] += sum_p latents[b, c_in, p + tap] * dx[p, c_out],
    into a flat-buffer slot; bit-identical reruns"""
    be = Backend(backend)
    g = torch.Generator().manual_seed(137 + b + c)
    m = b * h * w
    lat = rnd(g, b, 4, h, w).to(be.dev)
    dx = rnd(g, m, c).to(be.dev)
    prior = rnd(g, 36, c, scale=m ** 0.5)
    outs = []
    for _ in range(1 if be.emulated else 2):
        dw = FlatSlot(36, c, be.dev, prior)
        be.ops.conv_in_wgrad(lat, dx, dw.view.view(3, 3, 4, c), b, 4, h, w, c)
        be.sync()
        dw.check("conv_in_wgrad")
        outs.append(dw.view)
    ref, terms = _wgrad_ref(_rows(lat), dx, (b, h, w), 9)
    check_sum("dw", outs[0], ref, terms, old=prior.to(be.dev))
    if len(outs) > 1:
        assert torch.equal(outs[0], outs[1]), "two runs from the same prior differ"


# ------------------------------------------------------------------------------------------------ 4. optimizer ------
NORM_THREADS = 1056 * 256             # grad_sumsq's grid (optim.cu NORM_BLOCKS x 256 threads), one float4 per thread-step


def _tiny_params():
    from ddpo_b200.unet_spec import TINY, param_offsets
    return param_offsets(TINY)[1]


@pytest.mark.parametrize("backend,n", _backend_params(
    [(4,), (4 * NORM_THREADS - 4,), (4 * NORM_THREADS,), (4 * NORM_THREADS + 4,)], [(_tiny_params(),), (2 ** 26 + 4,)]))
def test_grad_sumsq(backend, n):
    """sum of squares of the flat gradient against an fp64 sum, at the grid-stride edge (one float4 short of, exactly
    at and one float4 past one float4 per thread), the TINY flat-buffer size and 2^26 + 4.  The last float4 holds a
    large share of the sum, so that dropping it cannot hide in the rounding."""
    be = Backend(backend)
    g = torch.Generator().manual_seed(139)
    x = rnd(g, n) * torch.exp(rnd(g, n))                      # magnitudes spread over several binades
    x[-4:] = torch.tensor([3.0, -5.0, 7.0, -11.0]) * max(1.0, (n / 4) ** 0.5)
    out = Guarded(1, 1, F32, be.dev, extra_rows=3)
    be.ops.grad_sumsq(x.to(be.dev), be.ops.optim_workspace(be.dev), out.view.reshape(1))
    be.sync()
    out.check("sumsq")
    ref = (x.double() ** 2).sum().item()
    # Every term is >= 0, so the error of a sum of depth d is at most gamma_d = d u / (1 - d u) of the sum
    # (u = 2^-24).  A term passes through: its square and two adds inside the float4 (3), the thread's running fp32
    # sum (k = ceil(n/4 / threads) steps), the 5 shuffle levels of warp_sum, the double-precision block and final sums
    # (counted as 1: their rounding is below 2^-24 of the sum) and the final cast to fp32 (1).
    k = -(-(n // 4) // NORM_THREADS)
    d = 3 + k + 5 + 1 + 1
    tol = d * U32 / (1 - d * U32)
    err = abs(out.view.item() - ref) / ref
    _record("sumsq", rel=err, bound=tol)
    assert err <= tol, f"relative error {err:.3g} (bound {tol:.3g}, depth {d})"


def _f32(v):
    return float(np.float32(v))


def _adamw_ref(p, acc, mu, nu, sumsq, hp, step):
    """float64 optax clip_by_global_norm + adamw (mu in bf16) step from the given fp32 / bf16 state, with the
    hyperparameters rounded to fp32 as the kernel receives them.  Returns the new state, the pre-rounding mu, the
    update ratio mu_hat / (sqrt(nu_hat) + eps), and the bounds of each output."""
    lr, b1, b2, eps, wd, gs, mn = (_f32(hp[k]) for k in ("lr", "b1", "b2", "eps", "wd", "grad_scale", "max_norm"))
    p, acc, mu, nu = p.double(), acc.double(), mu.double(), nu.double()
    norm = gs * float(sumsq) ** 0.5
    gr = acc * gs
    if not norm < mn:
        gr = gr / norm * mn
    mu_a, mu_b = (1 - b1) * gr, b1 * mu
    mu_new = mu_a + mu_b
    nu_new = (1 - b2) * gr * gr + b2 * nu
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    den = (nu_new / bc2).sqrt() + eps
    r = (mu_new / bc1) / den
    p_new = p - lr * (r + wd * p)
    # Rounding steps of clip_adamw_kernel, to first order in u = 2^-24 (each count rounded up):
    # - g~ = acc * scale (1); the clipped g^ = (g~ / norm) * max, norm = scale * sqrtf(sumsq) (2), / (1), * (1): <= 5u;
    # - mu = (1-b1) g^ + b1 mu_old ((1-b1) is exact in fp32): <= 7u of |(1-b1) g^| + |b1 mu_old|, counted as 8u;
    # - nu = (1-b2) g^2 + b2 nu_old, both terms >= 0: g^2 <= 11u, then the product and the add: <= 13u of nu, counted 16u;
    # - mu_hat = mu / bc1 (bc1 cast to fp32: 1, the division: 1); sqrt(nu / bc2) + eps: (16 + 2) / 2 + 1 + 1 <= 11u;
    #   r = mu_hat / den: the mu error, plus <= 14u of |r|; + wd p (2) -> u_ error <= e_mu / (bc1 den) + 14u |r| + 2u |wd p|;
    # - p + (-lr) u_: lr u_ (1), the add (1 of |p_new|).
    # mu is then stored as bf16: one more rounding of at most 2^-8 of its fp32 value.  That rounding reaches nearly the
    # whole 2^-8 for values just above a power of two, so the mu check is expected to use almost all of its bound.
    e_mu = 8 * U32 * (mu_a.abs() + mu_b.abs())
    b_nu = 16 * U32 * nu_new
    b_mu = U_BF16 * mu_new.abs() + (1 + U_BF16) * e_mu
    b_p = 2 * U32 * p_new.abs() + lr * (1.01 * e_mu / (bc1 * den) + 16 * U32 * (r.abs() + (wd * p).abs()))
    return dict(p=p_new, mu=mu_new, nu=nu_new, norm=norm, r=r), dict(p=b_p, mu=b_mu, nu=b_nu)


def _check_bounded(name, got, ref, bound):
    err = (got.double() - ref).abs()
    worst = (err / (bound + 1e-300)).max().item()
    _record(name, worst_over_bound=worst, max_abs=err.max().item())
    assert worst <= 1.0, f"{name}: error {worst:.3g} x its bound"


# (step, clipped): both branches of clip_by_global_norm, early steps where the bias corrections matter most, and late ones
ADAM_STEPS = [(1, True), (2, False), (3, True), (10, False), (1000, True)]


@pytest.mark.parametrize("backend,n", _backend_params([(4096,), (4 * NORM_THREADS + 4,)], [(_tiny_params(),)]))
def test_clip_adamw_consecutive_steps(backend, n):
    """clip_adamw over consecutive steps from a non-zero bf16 mu and fp32 nu, with grad_scale != 1 and wd > 0.  Each
    step's reference starts from the kernel's own state after the previous step, so errors do not compound; at steps > 1
    the old mu / nu and the bias corrections shape the update (at step 1 from zero state it is ~ sign(g))."""
    be = Backend(backend)
    g = torch.Generator().manual_seed(149)
    hp = dict(lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, wd=1e-2, grad_scale=0.25, max_norm=1.0)
    p = rnd(g, n).to(be.dev)
    mu = (rnd(g, n) * 1e-2).to(BF16).to(be.dev)
    nu = (rnd(g, n) * 1e-2).square().to(be.dev)
    norm_out = Guarded(1, 1, F32, be.dev, extra_rows=3)
    for step, clipped in ADAM_STEPS:
        target = 30.0 if clipped else 0.3                      # global norm of the scaled gradient / max_norm
        acc = rnd(g, n) * torch.exp(rnd(g, n) * 0.5)
        acc *= target * hp["max_norm"] / (hp["grad_scale"] * acc.double().norm().item())
        sumsq = torch.tensor([(acc.double() ** 2).sum().item()], dtype=F32)
        state = (p.clone(), acc.clone(), mu.clone(), nu.clone())
        acc = acc.to(be.dev)
        be.ops.clip_adamw(p, acc, mu, nu, sumsq.to(be.dev), hp["grad_scale"], hp["max_norm"], hp["lr"], hp["b1"],
                          hp["b2"], hp["eps"], hp["wd"], step, norm_out=norm_out.view.reshape(1))
        be.sync()
        ref, bound = _adamw_ref(state[0], state[1].to(be.dev), state[2], state[3], sumsq.item(), hp, step)
        assert (ref["norm"] >= hp["max_norm"]) == clipped
        _check_bounded(f"step{step} params", p, ref["p"], bound["p"])
        _check_bounded(f"step{step} nu", nu, ref["nu"], bound["nu"])
        _check_bounded(f"step{step} mu", mu, ref["mu"], bound["mu"])
        # norm = grad_scale * sqrtf(sumsq): two roundings
        assert abs(norm_out.view.item() - ref["norm"]) <= 2 * U32 * ref["norm"], "norm_out"
        norm_out.check("norm_out")
        assert torch.equal(acc, torch.zeros_like(acc)), "grad_acc is not zero after the step"
        # the update moved the parameters by much more than the bounds: the checks above are not vacuous
        assert (state[0].to(be.dev) - p).abs().max().item() > 100 * bound["p"].max().item()


@pytest.mark.parametrize("backend", _backend_params([()]))
def test_clip_adamw_matches_oracle_optimizer_over_steps(backend):
    """five clip_adamw steps against the NumPy restatement of the reference optimizer (oracle/optim.py), carrying the
    state across steps.  The two round in different orders, so their stored bf16 mu may land on neighbouring bf16
    values: each step adds at most 2^-7 (one bf16 unit in the last place) of |(1-b1) g| + |b1 mu_old| to the difference
    of the two mu, on top of b1 times the difference it inherits; a step's parameter update differs by lr times the mu
    difference over the bias-corrected denominator, plus d2 of the update (see below)."""
    from oracle import optim as OO
    be = Backend(backend)
    g = torch.Generator().manual_seed(151)
    n = 8192
    hp = dict(lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, wd=1e-2, max_norm=1.0)
    gs = 0.5
    p0 = rnd(g, n)
    p, mu, nu = p0.clone().to(be.dev), torch.zeros(n, dtype=BF16, device=be.dev), torch.zeros(n, device=be.dev)
    po, st = p0.numpy().copy(), OO.AdamWState(n)
    # clip_adamw receives b2 as fp32 and forms 1 - b2 from it; optax (and the oracle) round 1 - b2 to fp32.  The two
    # coefficients of g^2 differ by d2 (1.3e-5 of it at b2 = 0.999), so nu may differ by d2 of itself and the update,
    # through sqrt(nu), by d2 / 2 of itself
    d2 = abs((1 - _f32(hp["b2"])) - _f32(1 - hp["b2"])) / _f32(1 - hp["b2"])
    b1, b2 = hp["b1"], hp["b2"]
    mu_bnd, p_bnd = np.zeros(n), np.zeros(n)
    for step, target in enumerate((30.0, 0.3, 3.0, 0.5, 30.0), start=1):
        acc = rnd(g, n)
        acc *= target / (gs * acc.double().norm().item())
        sumsq = torch.tensor([(acc.double() ** 2).sum().item()], dtype=F32, device=be.dev)
        be.ops.clip_adamw(p, acc.clone().to(be.dev), mu, nu, sumsq, gs, hp["max_norm"], hp["lr"], b1, b2, hp["eps"],
                          hp["wd"], step)
        be.sync()
        gc = (acc * gs).double().numpy()
        gc = gc if target < hp["max_norm"] else gc / np.sqrt((gc ** 2).sum()) * hp["max_norm"]
        mu_old, prev = st.mu.astype(np.float64), po.astype(np.float64)
        po, _ = OO.clip_adamw_update(po, (acc * gs).numpy(), st, **hp)
        mu_bnd = 2 ** -7 * ((1 - b1) * np.abs(gc) + b1 * np.abs(mu_old)) + b1 * mu_bnd + 1e-12
        den = (1 - b1 ** step) * (np.sqrt(st.nu.astype(np.float64) / (1 - b2 ** step)) + hp["eps"])
        p_bnd += hp["lr"] * mu_bnd / den + (d2 + 64 * U32) * np.abs(po - prev)
        dp = np.abs(p.cpu().double().numpy() - po)
        worst = (dp / (p_bnd + 4 * U32 * np.abs(po))).max()
        _record(f"step{step} params", worst_over_bound=float(worst))
        assert worst <= 1.0, f"step {step}: params differ from the oracle by {worst:.3g} x the bound"
        dnu = np.abs(nu.cpu().double().numpy() - st.nu)
        assert (dnu <= (d2 + 64 * U32) * st.nu + 1e-30).all(), f"step {step}: nu differs from the oracle"
        dmu = np.abs(mu.cpu().double().numpy() - st.mu)
        assert (dmu <= mu_bnd).all(), f"step {step}: mu differs from the oracle"
        # the bounds are small against what a step does
        assert p_bnd.max() < 0.05 * step * hp["lr"]
