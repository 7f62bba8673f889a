"""GPU parity tests of the backward kernels (wgrad, norm backward, ...) vs torch autograd."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def bf(x):
    return x.to(torch.bfloat16)


@pytest.mark.parametrize("m,k,n", [(256, 64, 64), (1000, 320, 320), (4096, 1280, 640), (154, 1024, 1280), (8192, 128, 960),
                                   (5000, 192, 192), (40960, 320, 2560)])
def test_wgrad_linear(m, k, n):
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(0)
    x = bf(torch.randn(m, k, generator=g)).to(DEV)
    # dY is a column slice of a wider buffer (as the q/k/v gradients are): columns beyond n must not leak in
    dyw = bf(torch.randn(m, n + 64, generator=g)).to(DEV)
    dy = dyw[:, :n]
    dw = torch.ones(k, n, device=DEV)
    ops.wgrad(dy=dy, ldy=n + 64, n=n, x0=x, c0=k, m=m, dw=dw)
    torch.cuda.synchronize()
    ref = 1.0 + x.float().t() @ dy.float()
    err = (dw - ref).abs().max().item()
    assert err < 2e-3 * ref.abs().max().item(), f"max err {err}"


@pytest.mark.parametrize("b,h,c0,c1,n,ks,stride", [(2, 8, 64, 0, 64, 3, 1), (2, 16, 128, 64, 128, 3, 1), (4, 64, 64, 0, 64, 3, 1),
                                                   (2, 32, 320, 0, 320, 3, 1), (2, 16, 64, 64, 128, 1, 1),
                                                   (2, 8, 64, 0, 64, 3, 2), (3, 4, 64, 0, 64, 3, 1),
                                                   (2, 16, 320, 640, 320, 3, 1), (1, 8, 192, 0, 448, 3, 1)])
def test_wgrad_conv(b, h, c0, c1, n, ks, stride):
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(1)
    hi = h * stride
    x0 = bf(torch.randn(b, hi, hi, c0, generator=g)).to(DEV)
    x1 = bf(torch.randn(b, hi, hi, c1, generator=g)).to(DEV) if c1 else None
    dy = bf(torch.randn(b * h * h, n, generator=g)).to(DEV)
    cin = c0 + c1
    dw = torch.zeros(ks * ks * cin, n, device=DEV)
    ops.wgrad(dy=dy, n=n, x0=x0, x1=x1, c0=c0, c1=c1, conv=(b, h, h), taps=ks * ks, stride=stride, dw=dw)
    torch.cuda.synchronize()
    xin = (x0.float() if x1 is None else torch.cat([x0.float(), x1.float()], -1)).permute(0, 3, 1, 2).requires_grad_(False)
    w = torch.zeros(n, cin, ks, ks, device=DEV, requires_grad=True)
    y = torch.nn.functional.conv2d(xin, w, stride=stride, padding=ks // 2)
    y.backward(dy.float().view(b, h, h, n).permute(0, 3, 1, 2))
    ref = w.grad.permute(2, 3, 1, 0).reshape(ks * ks * cin, n)  # OIHW -> HWIO
    err = (dw - ref).abs().max().item()
    assert err < 2e-3 * max(1.0, ref.abs().max().item()), f"max err {err}"


@pytest.mark.parametrize("dy_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("b,hw,c0,c1,silu", [(2, 64, 64, 0, True), (2, 1024, 320, 0, True), (2, 256, 128, 64, False),
                                             # SD2-base up-block resnets: cin = 2560, 1920, 960, 640
                                             (2, 64, 1280, 1280, True), (2, 256, 1280, 640, True),
                                             (2, 1024, 640, 320, True), (2, 4096, 320, 320, True)])
def test_groupnorm_bwd(b, hw, c0, c1, silu, dy_dtype):
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(2)
    c = c0 + c1
    x0 = (torch.randn(b, hw, c0, generator=g) * 2 + 0.5).to(DEV)
    x1 = torch.randn(b, hw, c1, generator=g).to(DEV) if c1 else None
    sc = (1 + 0.1 * torch.randn(c, generator=g)).to(DEV)
    bi = (0.1 * torch.randn(c, generator=g)).to(DEV)
    dy_in = torch.randn(b, hw, c, generator=g).to(DEV).to(dy_dtype)   # bf16: what a dgrad GEMM hands to the norm's backward
    dy = dy_in.float()
    ws = torch.zeros(ops.groupnorm_workspace_floats(b, hw, c), device=DEV)
    y = torch.zeros(b, hw, c, dtype=torch.bfloat16, device=DEV)
    ops.groupnorm_fwd(x0, sc, bi, ws, b, hw, c0, x1=x1, c1=c1, silu=silu, y_bf16=y)
    dx0 = torch.zeros(b, hw, c0, device=DEV)
    dx1 = torch.zeros(b, hw, c1, device=DEV) if c1 else None
    dsc = torch.zeros(c, device=DEV)
    dbi = torch.zeros(c, device=DEV)
    ops.groupnorm_bwd(x0, sc, bi, ws, b, hw, c0, dy_in, dx0, dsc, dbi, x1=x1, c1=c1, dx1=dx1, silu=silu)
    torch.cuda.synchronize()
    x = (x0 if x1 is None else torch.cat([x0, x1], -1)).clone().requires_grad_(True)
    scr, bir = sc.clone().requires_grad_(True), bi.clone().requires_grad_(True)
    ref = torch.nn.functional.group_norm(x.permute(0, 2, 1), 32, scr, bir, 1e-5).permute(0, 2, 1)
    if silu:
        ref = torch.nn.functional.silu(ref)
    ref.backward(dy)
    gx = x.grad
    assert (dx0 - gx[..., :c0]).abs().max().item() < 2e-3 * gx.abs().max().item()
    if c1:
        assert (dx1 - gx[..., c0:]).abs().max().item() < 2e-3 * gx.abs().max().item()
    assert (dsc - scr.grad).abs().max().item() < 2e-3 * scr.grad.abs().max().item()
    assert (dbi - bir.grad).abs().max().item() < 2e-3 * bir.grad.abs().max().item()


@pytest.mark.parametrize("dy_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("m,c", [(64, 64), (1000, 320), (2048, 1280)])
def test_layernorm_bwd(m, c, dy_dtype):
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(3)
    x = (torch.randn(m, c, generator=g) * 3 + 1).to(DEV)
    sc = (1 + 0.1 * torch.randn(c, generator=g)).to(DEV)
    bi = (0.1 * torch.randn(c, generator=g)).to(DEV)
    dy_in = torch.randn(m, c, generator=g).to(DEV).to(dy_dtype)
    dy = dy_in.float()
    y = torch.zeros(m, c, dtype=torch.bfloat16, device=DEV)
    st = torch.zeros(m, 2, device=DEV)
    ops.layernorm_fwd(x, sc, bi, y, m, c, stats=st)
    dx = torch.ones(m, c, device=DEV)
    dsc = torch.zeros(c, device=DEV)
    dbi = torch.zeros(c, device=DEV)
    ws = torch.zeros(ops.layernorm_bwd_workspace_floats(m, c), device=DEV)
    ops.layernorm_bwd(x, sc, st, dy_in, dx, dsc, dbi, ws, m, c, accumulate=True)
    torch.cuda.synchronize()
    xr, scr, bir = x.clone().requires_grad_(True), sc.clone().requires_grad_(True), bi.clone().requires_grad_(True)
    torch.nn.functional.layer_norm(xr, (c,), scr, bir, 1e-5).backward(dy)
    assert (dx - 1.0 - xr.grad).abs().max().item() < 2e-3 * xr.grad.abs().max().item()
    assert (dsc - scr.grad).abs().max().item() < 2e-3 * scr.grad.abs().max().item()
    assert (dbi - bir.grad).abs().max().item() < 2e-3 * bir.grad.abs().max().item()


@pytest.mark.parametrize("b,heads,nq,nk", [(1, 1, 128, 128), (2, 2, 256, 256), (1, 2, 1024, 1024), (2, 2, 256, 77),
                                           (2, 3, 64, 64), (2, 1, 64, 77)])
def test_attention_bwd(b, heads, nq, nk):
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(4)
    c = heads * 64
    q = bf(torch.randn(b, nq, c, generator=g)).to(DEV)
    kv = bf(torch.randn(b, nk, 2 * c, generator=g)).to(DEV)
    do = bf(torch.randn(b, nq, c, generator=g)).to(DEV)
    out = torch.zeros(b, nq, c, dtype=torch.bfloat16, device=DEV)
    lse = torch.zeros(b, heads, nq, device=DEV)
    ops.attention_fwd(q, kv, kv[:, :, c:], out, b, heads, nq, nk, c, 2 * c, 2 * c, c, lse=lse)
    dq = torch.zeros(b, nq, c, dtype=torch.bfloat16, device=DEV)
    dkv = torch.zeros(b, nk, 2 * c, dtype=torch.bfloat16, device=DEV)
    delta = torch.zeros(b, heads, nq, device=DEV)
    ops.attention_bwd(q, kv, kv[:, :, c:], out, do, lse, delta, dq, dkv, dkv[:, :, c:], b, heads, nq, nk, c, 2 * c, 2 * c,
                      c, c, c, 2 * c, 2 * c)
    torch.cuda.synchronize()
    qr = q.float().requires_grad_(True)
    kvr = kv.float().requires_grad_(True)
    qh = qr.view(b, nq, heads, 64).permute(0, 2, 1, 3)
    kh = kvr[:, :, :c].reshape(b, nk, heads, 64).permute(0, 2, 1, 3)
    vh = kvr[:, :, c:].reshape(b, nk, heads, 64).permute(0, 2, 1, 3)
    o = (torch.softmax((qh @ kh.transpose(-1, -2)) * 0.125, dim=-1) @ vh).permute(0, 2, 1, 3).reshape(b, nq, c)
    o.backward(do.float())

    def rel(a, r):
        return ((a.float() - r).norm() / (r.norm() + 1e-12)).item()
    assert rel(dq, qr.grad) < 2e-2, f"dq {rel(dq, qr.grad)}"
    assert rel(dkv[:, :, :c], kvr.grad[:, :, :c]) < 2e-2, f"dk {rel(dkv[:, :, :c], kvr.grad[:, :, :c])}"
    assert rel(dkv[:, :, c:], kvr.grad[:, :, c:]) < 2e-2, f"dv {rel(dkv[:, :, c:], kvr.grad[:, :, c:])}"


# ---- stem convolutions (conv_in weight grad; conv_out dgrad + wgrad + dbias) vs torch autograd on the CPU ----
@pytest.mark.parametrize("b,h,w,c", [(2, 16, 16, 64), (3, 8, 24, 320), (1, 5, 7, 96)])
def test_conv_out_bwd(b, h, w, c):
    from ddpo_b200 import ops
    g = torch.Generator().manual_seed(b * 100 + c)
    x = torch.randn(b, h, w, c, generator=g)                 # NHWC fp32 (conv_out input)
    wt = torch.randn(3, 3, c, 4, generator=g) * 0.1          # HWIO
    dy = torch.randn(b, 4, h, w, generator=g)                # NCHW
    xr, wr = x.clone().requires_grad_(), wt.clone().requires_grad_()
    bias = torch.zeros(4, requires_grad=True)
    y = torch.nn.functional.conv2d(xr.permute(0, 3, 1, 2), wr.permute(3, 2, 0, 1), bias, padding=1)
    y.backward(dy)
    dx = torch.empty(b, h, w, c, device=DEV)
    dw = torch.ones(3, 3, c, 4, device=DEV)                  # kernels accumulate into the gradient buffers
    db = torch.ones(4, device=DEV)
    ops.conv_out_bwd(x.to(DEV), wt.to(DEV), dy.to(DEV), dx, dw, db, b, h, w, c)
    torch.cuda.synchronize()
    assert torch.allclose(dx.cpu(), xr.grad, rtol=1e-4, atol=1e-4)
    assert torch.allclose(dw.cpu() - 1, wr.grad, rtol=1e-4, atol=2e-3)
    assert torch.allclose(db.cpu() - 1, bias.grad, rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("b,h,w,c", [(2, 16, 16, 64), (3, 8, 24, 320), (1, 5, 7, 96)])
def test_conv_in_wgrad(b, h, w, c):
    from ddpo_b200 import ops
    g = torch.Generator().manual_seed(b * 10 + c)
    lat = torch.randn(b, 4, h, w, generator=g)               # NCHW latents
    dx = torch.randn(b, h, w, c, generator=g)                # NHWC gradient of the conv_in output
    wr = torch.zeros(3, 3, 4, c, requires_grad=True)         # HWIO
    y = torch.nn.functional.conv2d(lat, wr.permute(3, 2, 0, 1), None, padding=1)
    y.backward(dx.permute(0, 3, 1, 2))
    dw = torch.full((3, 3, 4, c), 2.0, device=DEV)
    ops.conv_in_wgrad(lat.to(DEV), dx.to(DEV), dw, b, 4, h, w, c)
    dw2 = torch.full((3, 3, 4, c), 2.0, device=DEV)
    ops.conv_in_wgrad(lat.to(DEV), dx.to(DEV), dw2, b, 4, h, w, c)
    torch.cuda.synchronize()
    assert torch.allclose(dw.cpu() - 2, wr.grad, rtol=1e-4, atol=2e-3)
    assert torch.equal(dw, dw2)                              # fixed reduction order -> bit-reproducible


@pytest.mark.parametrize("m,c", [(300, 64), (4096, 320)])
def test_geglu_bwd(m, c):
    """d(lin * gelu_tanh(gate)) from the tile-interleaved bf16 pre-activation the forward GEMM saved (bn = 256:
    [128 lin | 128 gate] per 256 columns) -> plain [lin(4c) | gate(4c)] bf16 gradient."""
    from ddpo_b200 import ops
    g = torch.Generator().manual_seed(5)
    n = 8 * c
    lin = bf(torch.randn(m, 4 * c, generator=g))
    gate = bf(torch.randn(m, 4 * c, generator=g))
    dff = torch.randn(m, 4 * c, generator=g)
    pre = torch.empty(m, n, dtype=torch.bfloat16)
    for t in range(n // 256):
        pre[:, t * 256:t * 256 + 128] = lin[:, t * 128:(t + 1) * 128]
        pre[:, t * 256 + 128:(t + 1) * 256] = gate[:, t * 128:(t + 1) * 128]
    lr, gr = lin.float().requires_grad_(), gate.float().requires_grad_()
    (lr * torch.nn.functional.gelu(gr, approximate="tanh")).backward(dff)
    dpre = torch.empty(m, n, dtype=torch.bfloat16, device=DEV)
    ops.geglu_bwd(pre.to(DEV), dff.to(DEV), dpre, m, n, 256)
    torch.cuda.synchronize()
    out = dpre.float().cpu()
    assert torch.allclose(out[:, :4 * c], lr.grad, rtol=1e-2, atol=1e-2)
    assert torch.allclose(out[:, 4 * c:], gr.grad, rtol=1e-2, atol=1e-2)
    # bf16 upstream gradient (what the FF down-projection's dgrad GEMM writes): same result as fp32 of the rounded values
    dpre2 = torch.empty(m, n, dtype=torch.bfloat16, device=DEV)
    ops.geglu_bwd(pre.to(DEV), bf(dff).to(DEV), dpre2, m, n, 256)
    dpre3 = torch.empty(m, n, dtype=torch.bfloat16, device=DEV)
    ops.geglu_bwd(pre.to(DEV), bf(dff).float().to(DEV), dpre3, m, n, 256)
    torch.cuda.synchronize()
    assert torch.equal(dpre2, dpre3)
