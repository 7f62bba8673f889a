"""TEST INFRASTRUCTURE: a torch-CPU emulation of the handful of ``ddpo_b200.ops`` entry points the VAE decoder
sequences, with the same argument conventions (bf16 operands, fp32 accumulation, [N, K] weights, NHWC).  It lets the
CPU suite dry-run the HOST-side assembly of ``ddpo_b200/vae.py`` (buffer shapes, operand order, bias / residual
plumbing, chunking) against the oracle without a GPU.  It is never imported by the package: the product path has no
CPU fallback (``ops._p`` asserts CUDA tensors)."""
import torch
import torch.nn.functional as F

BF16, F32 = torch.bfloat16, torch.float32


class CpuArena:
    def __init__(self, device=None):
        self.total_bytes = 0

    def alloc(self, shape, dtype):
        return torch.zeros(*shape, dtype=dtype)

    def alloc_with_gn_stats(self, shape, hw):
        t = self.alloc(shape, torch.float32)
        # NaN-filled: a GroupNorm that reads statistics nobody wrote fails loudly
        t._gn_stats = torch.full(gn_stats_shape(shape[0], shape[1]), float("nan")) if hw % 32 == 0 else None
        return t

    def release(self, t):
        pass


def groupnorm_workspace_floats(batch, hw, channels):
    return 8


def prep_weight(src, dst, k, n, ldk=None, row_offset=0, col_offset=0, geglu_bn=0):
    dst[row_offset:row_offset + n, :k].copy_(src.reshape(k, n).t().to(BF16))


def gn_stats_shape(rows, channels):
    return ((int(rows) + 31) // 32, int(channels), 2)


def _fill_gn_stats(gn_stats, y):
    """what the igemm epilogue leaves for the consuming GroupNorm: per 32-row slab and column (sum, sum of squares)"""
    rows, n = y.shape
    pad = (-rows) % 32
    yp = torch.cat([y, y.new_zeros(pad, n)]) if pad else y
    t = yp.reshape(-1, 32, n)
    gn_stats.copy_(torch.stack([t.sum(1), (t * t).sum(1)], -1))


def groupnorm_fwd(x0, scale, bias, ws, batch, hw, c0, x1=None, c1=0, silu=True, y_bf16=None, y_f32=None, raw_bf16=None,
                  skip_stats=False, eps=1e-5, stats0=None, stats1=None):
    assert x1 is None
    x = x0.reshape(batch, hw, 32, c0 // 32).float()
    if stats0 is not None and hw % 32 == 0:
        # the product takes mean / variance from the producer's slab statistics: do the same, so that a wrong or stale
        # statistics buffer handed over by the host code shows up in the CPU dry runs
        st = stats0.reshape(batch, hw // 32, 32, c0 // 32, 2).sum(dim=(1, 3))
        cnt = hw * (c0 // 32)
        mean = (st[..., 0] / cnt).reshape(batch, 1, 32, 1)
        var = ((st[..., 1] / cnt).reshape(batch, 1, 32, 1) - mean * mean).clamp(min=0)
    else:
        mean = x.mean(dim=(1, 3), keepdim=True)
        var = ((x * x).mean(dim=(1, 3), keepdim=True) - mean * mean).clamp(min=0)
    y = ((x - mean) * torch.rsqrt(var + eps)).reshape(batch * hw, c0) * scale + bias
    if silu:
        y = y * torch.sigmoid(y)
    if y_bf16 is not None:
        y_bf16.copy_(y.to(BF16))
    if y_f32 is not None:
        y_f32.copy_(y)
    if raw_bf16 is not None:
        raw_bf16.copy_(x0.reshape(batch * hw, c0).to(BF16))


def conv_in(x_nchw, w, bias, y_nhwc, batch, cin, h, wd, cout, gn_stats=None):
    assert cin <= 8 and cout % 4 == 0
    y = F.conv2d(x_nchw, w.permute(3, 2, 0, 1), bias, padding=1).permute(0, 2, 3, 1)
    y_nhwc.reshape(batch, h, wd, cout).copy_(y)
    if gn_stats is not None:
        _fill_gn_stats(gn_stats, y.reshape(batch * h * wd, cout))


def vae_post_quant(latents, w, bias, out, scaling=0.18215):
    out.copy_(torch.einsum("bihw,io->bohw", latents / scaling, w.reshape(4, 4)) + bias[None, :, None, None])


def upsample2x_bf16(x, y, batch, h, w, c):
    v = x.reshape(batch, h, w, c).repeat_interleave(2, 1).repeat_interleave(2, 2)
    y.reshape(batch, 2 * h, 2 * w, c).copy_(v.to(BF16))


def softmax_rows(scores, probs_bf16, scale):
    probs_bf16.copy_(torch.softmax(scores * scale, -1).to(BF16))


def image_to_uint8(img, out_u8):
    out_u8.copy_((img * 255).to(torch.uint8))


def vae_image_to_nchw(img_nhwc, out_nchw):
    out_nchw.copy_(((img_nhwc - 0.5) / 0.5).permute(0, 3, 1, 2))


def vae_encoder_head(x_nhwc, w, bias, wq, bq, moments, batch, h, wd, cin):
    hcv = F.conv2d(x_nhwc.reshape(batch, h, wd, cin).permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), bias, padding=1)
    m = torch.einsum("bihw,io->bhwo", hcv, wq.reshape(8, 8)) + bq
    moments.copy_(torch.cat([m[..., :4], m[..., 4:].clamp(-30.0, 20.0)], -1))


def vae_conv_out(x_nhwc, w, bias, batch, h, wd, cin, raw_nchw=None, img_nhwc=None):
    raw = F.conv2d(x_nhwc.reshape(batch, h, wd, cin).permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), bias, padding=1)
    if raw_nchw is not None:
        raw_nchw.copy_(raw)
    if img_nhwc is not None:
        img_nhwc.copy_((raw / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1))


# ---- text encoder ----
def embed_tokens(ids, token_embedding, position_embedding, out, seq_len):
    rows = ids.numel()
    pos = position_embedding[torch.arange(rows) % seq_len]
    out.copy_(token_embedding[ids.long()] + pos)


def layernorm_fwd(x, scale, bias, y_bf16, m, c, stats=None):
    xf = x.reshape(m, c).float()
    mean = xf.mean(-1, keepdim=True)
    var = ((xf * xf).mean(-1, keepdim=True) - mean * mean).clamp(min=0)
    y_bf16.reshape(m, c).copy_(((xf - mean) * torch.rsqrt(var + 1e-5) * scale + bias).to(BF16))


def layernorm_f32(x, scale, bias, y, m, c, eps=1e-5):
    xf = x.reshape(m, c).float()
    mean = xf.mean(-1, keepdim=True)
    var = ((xf * xf).mean(-1, keepdim=True) - mean * mean).clamp(min=0)
    y.reshape(m, c).copy_((xf - mean) * torch.rsqrt(var + eps) * scale + bias)


def act_bf16(x, y_bf16, act):
    y = x * torch.sigmoid(1.702 * x) if act == "quick_gelu" else F.gelu(x)
    y_bf16.copy_(y.to(BF16))


def attention_fwd(q, k, v, out, batch, heads, nq, nk, ldq, ldk, ldv, ldo, lse=None, causal=False):
    """q/k/v are column-offset VIEWS of a [rows, ld] bf16 matrix, head h at columns [h*64, h*64+64)."""
    def heads_of(t, n):
        return t[:, : heads * 64].reshape(batch, n, heads, 64).permute(0, 2, 1, 3).float()
    qq, kk, vv = heads_of(q, nq), heads_of(k, nk), heads_of(v, nk)
    s = qq @ kk.transpose(-1, -2) * (64 ** -0.5)
    if causal:
        s = s + torch.full((nq, nk), float("-inf")).triu(1)
    p = torch.softmax(s, -1).to(BF16).float()           # the kernel rounds P to bf16 before P V
    o = (p @ vv).permute(0, 2, 1, 3).reshape(batch * nq, heads * 64)
    out[:, : heads * 64].copy_(o.to(BF16))


# ---- image tower ----
def patchify_bf16(img_nhwc, out_bf16, patch):
    b, s, _, _ = img_nhwc.shape
    n = s // patch
    pt = img_nhwc.reshape(b, n, patch, n, patch, 3).permute(0, 1, 3, 2, 4, 5).reshape(b * n * n, patch * patch * 3)
    out_bf16.zero_()
    out_bf16[:, : pt.shape[1]].copy_(pt.to(BF16))


def vit_tokens(patches, class_embedding, position_embedding, out, batch, n_patches, dim):
    tok = torch.cat([class_embedding.expand(batch, 1, dim), patches.reshape(batch, n_patches, dim)], 1) + position_embedding[None]
    out.copy_(tok.reshape(batch * (n_patches + 1), dim))


def l2norm_rows(x, y):
    y.copy_(x / x.norm(dim=-1, keepdim=True))


def gather_rows(src, index, dst):
    dst.copy_(src.reshape(-1, dst.shape[-1])[index.long()].reshape(dst.shape))


# ---- U-Net forward (sampling path) ----
import math  # noqa: E402

import numpy as np  # noqa: E402


def _geglu_row(n_idx, N, bn):
    half, hn = bn >> 1, N >> 1
    j = n_idx if n_idx < hn else n_idx - hn
    return (j // half) * bn + (0 if n_idx < hn else half) + (j % half)


_prep_weight_plain = prep_weight


def prep_weight(src, dst, k, n, ldk=None, row_offset=0, col_offset=0, geglu_bn=0):  # noqa: F811
    if not geglu_bn:
        return _prep_weight_plain(src, dst, k, n, ldk, row_offset, col_offset, 0)
    rows = torch.tensor([_geglu_row(i, n, geglu_bn) for i in range(n)])
    dst[rows + row_offset, col_offset:col_offset + k] = src.reshape(k, n).t().to(BF16)


def permute_geglu_bias(src, dst, n, bn):
    rows = torch.tensor([_geglu_row(i, n, bn) for i in range(n)])
    dst[rows] = src


def cast_bf16(x, y):
    y.copy_(x.reshape(y.shape).to(BF16))


def timestep_sincos(t, out, batch, dim):
    half = dim // 2
    f = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000.0) / half))
    tt = t.float().reshape(-1)
    tt = tt.expand(batch) if tt.numel() == 1 else tt
    a = tt[:, None] * f[None]
    out.copy_(torch.cat([torch.cos(a), torch.sin(a)], 1))


_silu = lambda v: v * torch.sigmoid(v)


def dense_small(x, w, bias, y, batch, k, n, silu_in=False, silu_out=False):
    xv = x.reshape(batch, k)
    r = (_silu(xv) if silu_in else xv) @ w.reshape(k, n) + (bias if bias is not None else 0)
    y.copy_(_silu(r) if silu_out else r)


def dense_small_group_table(entries, device):
    rec, cta = [], 0
    for (w_off, b_off, y_off, n) in entries:
        rec.append((w_off, b_off, y_off, n, cta))
        cta += (n + 31) // 32
    return rec, cta


def dense_small_grouped(x, params_base, y_base, table, n_groups, total_ctas, batch, k):
    assert len(table) == n_groups and table[-1][4] + (table[-1][3] + 31) // 32 == total_ctas
    for (w_off, b_off, y_off, n, _) in table:
        w = params_base[w_off:w_off + k * n].reshape(k, n)
        y_base[y_off:y_off + batch * n].reshape(batch, n).copy_(x.reshape(batch, k) @ w + params_base[b_off:b_off + n])


_groupnorm_single = groupnorm_fwd


def groupnorm_fwd(x0, scale, bias, ws, batch, hw, c0, x1=None, c1=0, silu=True, y_bf16=None, y_f32=None,  # noqa: F811
                  raw_bf16=None, skip_stats=False, eps=1e-5, stats0=None, stats1=None):
    if x1 is None:
        return _groupnorm_single(x0, scale, bias, ws, batch, hw, c0, None, 0, silu, y_bf16, y_f32, raw_bf16, skip_stats, eps,
                                 stats0)
    cat = torch.cat([x0.reshape(batch * hw, c0), x1.reshape(batch * hw, c1)], 1)
    st = torch.cat([stats0, stats1], 1) if stats0 is not None and stats1 is not None else None
    return _groupnorm_single(cat, scale, bias, ws, batch, hw, c0 + c1, None, 0, silu, y_bf16, y_f32, raw_bf16, skip_stats, eps,
                             st)


def igemm(*, a0, wt, n, a1=None, c0=None, c1=0, lda0=None, lda1=None, conv=None, m=None, taps=1, stride=1, bias=None,
          rowvec=None, rows_per_sample=0, rowvec_ld=0, residual=None, ld_res=0, out_f32=None, out_bf16=None, ld_out=0,
          geglu=False, accumulate=False, bn=0, aux_bf16=None, gn_stats=None, no_low_pad=False):
    assert a0.dtype == BF16 and wt.dtype == BF16 and (a1 is None or a1.dtype == BF16)
    if conv is None and a0.dim() == 2 and c0 is not None and a0.shape[1] != c0:
        a0 = a0[:, :c0].contiguous()     # a column-offset view of a wider matrix as the linear A operand (lda0 = its pitch)
    c0 = int(c0 if c0 is not None else a0.shape[-1])
    cin = c0 + c1
    assert c0 % 64 == 0 and c1 % 64 == 0 and n % 32 == 0, (c0, c1, n)
    w = wt.reshape(n, taps * cin).float()
    if conv is not None:
        b, h, wd = conv
        hi, wi = h * stride, wd * stride
        x = a0.reshape(b, hi, wi, c0).float()
        if a1 is not None:
            x = torch.cat([x, a1.reshape(b, hi, wi, c1).float()], -1)
        ks = 3 if taps == 9 else 1
        wk = w.reshape(n, ks, ks, cin).permute(0, 3, 1, 2)
        if no_low_pad:      # pad on the high side only, then VALID (the VAE encoder's down-sample)
            y = F.conv2d(F.pad(x.permute(0, 3, 1, 2), (0, 1, 0, 1)), wk, None, stride=stride)
        else:
            y = F.conv2d(x.permute(0, 3, 1, 2), wk, None, stride=stride, padding=ks // 2)
        y = y.permute(0, 2, 3, 1).reshape(b * h * wd, n)
    else:
        assert taps == 1 and a1 is None
        y = a0.reshape(m, c0).float() @ w.t()
    if bias is not None:
        y = y + bias.reshape(1, n)
    if rowvec is not None:
        rv = rowvec.reshape(-1, rowvec_ld)[:, :n]
        y = (y.reshape(rv.shape[0], rows_per_sample, n) + rv[:, None]).reshape(-1, n)
    if geglu:
        assert bn and residual is None
        if aux_bf16 is not None:
            aux_bf16.reshape(y.shape).copy_(y.to(BF16))
        t = y.reshape(y.shape[0], n // bn, 2, bn // 2)
        lin, gate = t[:, :, 0], t[:, :, 1]
        act = lin * 0.5 * gate * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (gate + 0.044715 * gate ** 3)))
        out_bf16.reshape(y.shape[0], n // 2).copy_(act.reshape(y.shape[0], n // 2).to(BF16))
        return
    if residual is not None:
        y = y + residual.reshape(y.shape)
    if out_f32 is not None:
        out_f32.reshape(y.shape).copy_(out_f32.reshape(y.shape) + y if accumulate else y)
    if out_bf16 is not None:
        out_bf16.reshape(y.shape).copy_(y.to(BF16))
    if gn_stats is not None:
        assert out_f32 is not None and not accumulate
        _fill_gn_stats(gn_stats, y)


def conv_out(x_nhwc, w, bias, y_nchw, batch, h, wd, cin, cout):
    y_nchw.copy_(F.conv2d(x_nhwc.reshape(batch, h, wd, cin).permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), bias, padding=1))


# ---- U-Net backward (training path).  Gradient ops are emulated with torch autograd of the emulated forward op ----
def prep_weight_dgrad(src, dst, taps, k, n, ld_dst=0, col_offset=0):
    s = src.reshape(taps, k, n)
    ld = ld_dst or taps * n
    dst.reshape(k, ld)[:, col_offset:col_offset + taps * n].copy_(s.flip(0).permute(1, 0, 2).reshape(k, taps * n).to(BF16))


def layernorm_bwd_workspace_floats(m, c):
    return 8


def copy2d(src, lds, dst, ldd, rows, cols, accumulate=False):
    s = src.reshape(rows, -1)[:, :cols]
    d = dst.reshape(rows, -1)
    d[:, :cols] = d[:, :cols] + s if accumulate else s


def colsum_cast(dy, m, n, y_bf16=None, out=None, rows_per_group=None, accumulate=True, ld=0):
    v = dy.reshape(m, -1)[:, :n].float()
    if y_bf16 is not None:
        y_bf16.reshape(m, -1)[:, :n] = v.to(BF16)
    if out is not None:
        rpg = int(rows_per_group or m)
        s = v.reshape(m // rpg, rpg, n).sum(1)
        out.reshape(m // rpg, n).copy_(out.reshape(m // rpg, n) + s if accumulate else s)


def colsum_bf16(x, m, n, out, accumulate=True, ld=0):
    s = x.reshape(m, -1)[:, :n].float().sum(0, keepdim=True)
    out.reshape(1, n).copy_(out.reshape(1, n) + s if accumulate else s)


def _patches(x_nhwc, taps, stride):
    """[B, Hi, Wi, C] -> [B*Ho*Wo, taps*C] in (tap, c) order (pad 1 for 3x3)"""
    b, hi, wi, c = x_nhwc.shape
    if taps == 1:
        return x_nhwc.reshape(-1, c)
    u = F.unfold(x_nhwc.permute(0, 3, 1, 2), 3, padding=1, stride=stride)         # [B, C*9, L], (c, ky, kx) order
    u = u.reshape(b, c, 9, -1).permute(0, 3, 2, 1).reshape(-1, 9 * c)
    return u


def wgrad(*, dy, n, x0, dw, x1=None, c0=None, c1=0, ldy=0, ldx0=0, ldx1=0, conv=None, m=None, taps=1, stride=1):
    c0 = int(c0 if c0 is not None else x0.shape[-1])
    if conv is not None:
        b, h, wd = conv
        x = x0.reshape(b, h * stride, wd * stride, -1)[..., :c0].float()
        if x1 is not None:
            x = torch.cat([x, x1.reshape(b, h * stride, wd * stride, -1)[..., :c1].float()], -1)
        rows = b * h * wd
        pt = _patches(x, taps, stride)
    else:
        rows = m
        pt = x0.reshape(m, -1)[:, :c0].float()
    g = dy.reshape(rows, -1)[:, :n].float()
    dw.reshape(pt.shape[1], n).add_(pt.t() @ g)


def upsample2x_bwd(dy, dx, batch, h, w, c, accumulate=False):
    s = dy.reshape(batch, h, 2, w, 2, c).sum(dim=(2, 4)).reshape(batch * h * w, c)
    dx.reshape(batch * h * w, c).copy_(dx.reshape(batch * h * w, c) + s if accumulate else s)


def dilate2x_bf16(x, y, batch, h, w, c):
    out = torch.zeros(batch, 2 * h, 2 * w, c, dtype=BF16)
    out[:, ::2, ::2] = x.reshape(batch, h, w, c).to(BF16)
    y.reshape(out.shape).copy_(out)


def _gn_forward(x, scale, bias, batch, hw, c, silu, eps=1e-5):
    xg = x.reshape(batch, hw, 32, c // 32)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    var = ((xg * xg).mean(dim=(1, 3), keepdim=True) - mean * mean).clamp(min=0)
    y = ((xg - mean) * torch.rsqrt(var + eps)).reshape(batch * hw, c) * scale + bias
    return y * torch.sigmoid(y) if silu else y


def groupnorm_bwd(x0, scale, bias, ws, batch, hw, c0, dy, dx0, dscale, dbias, x1=None, c1=0, dx1=None, silu=True,
                  accumulate=False, ldd0=0, ldd1=0):
    m, c = batch * hw, c0 + c1
    x = x0.reshape(m, -1)[:, :c0]
    if x1 is not None:
        x = torch.cat([x, x1.reshape(m, -1)[:, :c1]], 1)
    x = x.detach().float().clone().requires_grad_(True)
    sc, bi = scale.detach().clone().requires_grad_(True), bias.detach().clone().requires_grad_(True)
    _gn_forward(x, sc, bi, batch, hw, c, silu).backward(dy.reshape(m, -1)[:, :c].float())
    dscale.add_(sc.grad)
    dbias.add_(bi.grad)
    d0 = dx0.reshape(m, -1)
    d0[:, :c0] = d0[:, :c0] + x.grad[:, :c0] if accumulate else x.grad[:, :c0]
    if x1 is not None:
        d1 = dx1.reshape(m, -1) if dx1.dim() != 2 else dx1
        d1[:, :c1] = d1[:, :c1] + x.grad[:, c0:] if accumulate else x.grad[:, c0:]


def layernorm_bwd(x, scale, stats, dy, dx, dscale, dbias, ws, m, c, accumulate=False):
    xv = x.reshape(m, c).detach().float().clone().requires_grad_(True)
    sc = scale.detach().clone().requires_grad_(True)
    bi = torch.zeros(c, requires_grad=True)
    mean = xv.mean(-1, keepdim=True)
    var = ((xv * xv).mean(-1, keepdim=True) - mean * mean).clamp(min=0)
    ((xv - mean) * torch.rsqrt(var + 1e-5) * sc + bi).backward(dy.reshape(m, c).float())
    dscale.add_(sc.grad)
    dbias.add_(bi.grad)
    d = dx.reshape(m, c)
    d.copy_(d + xv.grad if accumulate else xv.grad)


def geglu_bwd(pre, dff, dpre, m, n, bn=256):
    p = pre.reshape(m, n // bn, 2, bn // 2).float().detach().clone().requires_grad_(True)
    lin, gate = p[:, :, 0], p[:, :, 1]
    act = lin * 0.5 * gate * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (gate + 0.044715 * gate ** 3)))
    act.reshape(m, n // 2).backward(dff.reshape(m, n // 2).float())
    # the kernel reads the tile-interleaved pre-activation but writes the gradient in PLAIN order [lin(n/2) | gate(n/2)]
    gl, gg = p.grad[:, :, 0].reshape(m, n // 2), p.grad[:, :, 1].reshape(m, n // 2)
    dpre.reshape(m, n).copy_(torch.cat([gl, gg], 1).to(BF16))


def attention_bwd(q, k, v, out, dout, lse, delta, dq, dk, dv, batch, heads, nq, nk, ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv):
    def heads_of(t, n):
        return t[:, : heads * 64].reshape(batch, n, heads, 64).permute(0, 2, 1, 3).float().detach().clone().requires_grad_(True)
    qq, kk, vv = heads_of(q, nq), heads_of(k, nk), heads_of(v, nk)
    o = torch.softmax(qq @ kk.transpose(-1, -2) * (64 ** -0.5), -1) @ vv
    g = dout[:, : heads * 64].reshape(batch, nq, heads, 64).permute(0, 2, 1, 3).float()
    o.backward(g)
    back = lambda t, n: t.permute(0, 2, 1, 3).reshape(batch * n, heads * 64).to(BF16)
    dq[:, : heads * 64] = back(qq.grad, nq)
    dk[:, : heads * 64] = back(kk.grad, nk)
    dv[:, : heads * 64] = back(vv.grad, nk)


def conv_out_bwd(x_nhwc, w, dy_nchw, dx_nhwc, dw, dbias, batch, h, wd, cin):
    x = x_nhwc.reshape(batch, h, wd, cin).detach().float().clone().requires_grad_(True)
    wk = w.detach().clone().requires_grad_(True)
    bz = torch.zeros(w.shape[-1], requires_grad=True)
    F.conv2d(x.permute(0, 3, 1, 2), wk.permute(3, 2, 0, 1), bz, padding=1).backward(dy_nchw.reshape(batch, -1, h, wd).float())
    dx_nhwc.reshape(x.shape).copy_(x.grad)
    dw.add_(wk.grad)
    dbias.add_(bz.grad)


def conv_in_wgrad(lat, dx_nhwc, dw, batch, cin, h, wd, cout):
    wk = torch.zeros(3, 3, cin, cout, requires_grad=True)
    F.conv2d(lat.float(), wk.permute(3, 2, 0, 1), None, padding=1).backward(
        dx_nhwc.reshape(batch, h, wd, cout).permute(0, 3, 1, 2).float())
    dw.add_(wk.grad)


def dense_small_bwd(x, w, bias, dy, dpre_ws, dw, db, dx, batch, k, n, silu_in=False, silu_out=False, dx_accumulate=False):
    xv = x.reshape(batch, k).detach().float().clone().requires_grad_(True)
    wk = w.reshape(k, n).detach().clone().requires_grad_(True)
    bz = (bias.detach().clone() if bias is not None else torch.zeros(n)).requires_grad_(True)
    r = (_silu(xv) if silu_in else xv) @ wk + bz
    (_silu(r) if silu_out else r).backward(dy.reshape(batch, n).float())
    dw.reshape(k, n).add_(wk.grad)
    db.add_(bz.grad)
    if dx is not None:
        dx.reshape(batch, k).copy_(dx.reshape(batch, k) + xv.grad if dx_accumulate else xv.grad)


# ---- scheduler / PPO / optimizer ops (sampler + train_step dry runs); host-only helpers come from the real module ----
from ddpo_b200 import ops as _real_ops  # noqa: E402

prng_key, threefry_split, threefry_randint, key_tensor = (_real_ops.prng_key, _real_ops.threefry_split,
                                                          _real_ops.threefry_randint, _real_ops.key_tensor)


def _key_np(key_dev):
    return key_dev.reshape(-1)[:2].to(torch.int64).numpy().astype(np.int64).astype(np.uint64).astype(np.uint32)


def threefry_normal(key_dev, out):
    from oracle import threefry
    k = np.array([int(v) & 0xFFFFFFFF for v in key_dev.reshape(-1)[:2].tolist()], np.uint32)
    out.copy_(torch.from_numpy(threefry.normal(k, (out.numel(),))).reshape(out.shape))
    return out


def ddim_workspace(batch, device):
    return torch.zeros(batch * 9)


def optim_workspace(device):
    return torch.zeros(8, dtype=torch.uint8)


def _ddim_terms(eps_u, eps_c, sample, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta, pred="epsilon"):
    b = sample.shape[0]
    t = timesteps.reshape(-1).long()
    t = t.expand(b) if t.numel() == 1 else t
    pt = t - step_ratio
    a_t = alphas_cumprod[t]
    a_prev = torch.where(pt >= 0, alphas_cumprod[pt.clamp(min=0)], torch.tensor(float(final_alpha)))
    var = ((1 - a_prev) / (1 - a_t)) * (1 - a_t / a_prev)
    sigma = float(eta) * torch.sqrt(var)
    a_t, a_prev, sigma = a_t[:, None], a_prev[:, None], sigma[:, None]
    eps = eps_u + float(guidance) * (eps_c - eps_u)
    d = torch.sqrt(1 - a_prev - sigma ** 2)
    if pred == "epsilon":
        x0 = (sample - torch.sqrt(1 - a_t) * eps) / torch.sqrt(a_t)
        mean = torch.sqrt(a_prev) * x0 + d * eps
        c_eps = d - torch.sqrt(a_prev) * torch.sqrt(1 - a_t) / torch.sqrt(a_t)
    elif pred == "sample":
        c_eps = torch.sqrt(a_prev) + d
        mean = c_eps * eps
    else:
        x0 = torch.sqrt(a_t) * sample - torch.sqrt(1 - a_t) * eps
        mean = torch.sqrt(a_prev) * x0 + d * (torch.sqrt(a_t) * eps + torch.sqrt(1 - a_t) * sample)
        c_eps = d * torch.sqrt(a_t) - torch.sqrt(a_prev) * torch.sqrt(1 - a_t)
    return mean, sigma, sigma.clamp(min=1e-6), c_eps


def _logp(prev, mean, sd):
    return (-((prev - mean) ** 2) / (2 * sd ** 2) - torch.log(sd) - 0.9189385332046727).mean(1)


def ddim_step_sample(eps_u, eps_c, sample, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta, key_dev,
                     prev_out, logp_out, ws, pred="epsilon"):
    mean, sigma, sd, _ = _ddim_terms(eps_u, eps_c, sample, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta, pred)
    z = torch.empty_like(sample)
    threefry_normal(key_dev, z)
    prev_out.copy_(mean + sigma * z)
    logp_out.copy_(_logp(prev_out, mean, sd))


def ddim_logprob_fwd(eps_u, eps_c, sample, prev, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta,
                     logp_out, ws, pred="epsilon"):
    mean, _, sd, _ = _ddim_terms(eps_u, eps_c, sample, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta, pred)
    logp_out.copy_(_logp(prev, mean, sd))


def ddim_logprob_bwd(eps_u, eps_c, sample, prev, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta, dlogp,
                     d_eps_u, d_eps_c, ws, pred="epsilon"):
    mean, _, sd, c_eps = _ddim_terms(eps_u, eps_c, sample, alphas_cumprod, timesteps, final_alpha, step_ratio, guidance, eta, pred)
    k = (prev - mean) / sd ** 2 * c_eps * dlogp[:, None] / sample.shape[1]
    d_eps_c.copy_(float(guidance) * k)
    if d_eps_u is not None:
        d_eps_u.copy_((1.0 - float(guidance)) * k)


def ppo_loss(logp, old_logp, adv, clip_range, info_out, dlogp_out, micro_batch=None):
    from oracle import ppo
    n = logp.numel()
    loss, info, dlp = ppo.ppo_loss(logp.numpy(), old_logp.numpy(), adv.numpy(), clip_range)
    info_out.copy_(torch.tensor([float(info["approx_kl"]), float(info["clipfrac"]), float(info["loss"])]))
    dlogp_out.copy_(torch.from_numpy(dlp) * n / int(micro_batch or n))


def grad_sumsq(g, ws, out):
    out.copy_((g.double() ** 2).sum().float().reshape(1))


def clip_adamw(params, grad_acc, mu, nu, sumsq, grad_scale, max_norm, lr, b1, b2, eps, wd, step, norm_out=None):
    # the kernel receives the hyperparameters as fp32 and forms 1 - b1 and 1 - b2 from those (exact in fp32)
    lr, b1, b2, eps, wd = (float(np.float32(v)) for v in (lr, b1, b2, eps, wd))
    norm = float(grad_scale) * float(sumsq.sqrt())
    g = grad_acc * float(grad_scale)
    if not norm < max_norm:
        g = g / norm * max_norm
    m = (1 - b1) * g + b1 * mu.float()
    v = (1 - b2) * g * g + b2 * nu
    upd = (m / (1 - b1 ** step)) / (torch.sqrt(v / (1 - b2 ** step)) + eps) + wd * params
    params.add_(-lr * upd)
    mu.copy_(m.to(BF16))
    nu.copy_(v)
    grad_acc.zero_()
    if norm_out is not None:
        norm_out.fill_(norm)


# ---- RWR ops ----
def rwr_workspace(batch, device):
    return torch.zeros(batch * 10 + 1)


def rwr_noisy_latents(moments_nhwc, key_sample_dev, key_noise_dev, timesteps, alphas_cumprod, noise_out, noisy_out,
                      latents_out=None, scaling=0.18215):
    from oracle import threefry
    kk = lambda k: np.array([int(v) & 0xFFFFFFFF for v in k.reshape(-1)[:2].tolist()], np.uint32)
    mom = moments_nhwc.float()
    mean, logvar = mom.chunk(2, dim=-1)
    std = torch.exp(0.5 * logvar.clamp(-30.0, 20.0))
    z = torch.from_numpy(threefry.normal(kk(key_sample_dev), tuple(mean.shape)))
    lat = ((mean + std * z) * scaling).permute(0, 3, 1, 2)
    nz = torch.from_numpy(threefry.normal(kk(key_noise_dev), tuple(lat.shape)))
    a = alphas_cumprod[timesteps.long()].reshape(-1, 1, 1, 1)
    noise_out.copy_(nz)
    noisy_out.copy_(torch.sqrt(a) * lat + torch.sqrt(1 - a) * nz)
    if latents_out is not None:
        latents_out.copy_(lat)


def rwr_mse_loss(eps_u, eps_c, noise, guidance, loss_out, ws, weights=None, per_sample=None, d_eps_u=None, d_eps_c=None):
    b, n = noise.shape
    pred = eps_u + float(guidance) * (eps_c - eps_u)
    d = pred - noise
    per = (d * d).mean(1)
    w = weights if weights is not None else torch.full((b,), 1.0 / b)
    loss_out.copy_((per * w).sum().reshape(1))
    if per_sample is not None:
        per_sample.copy_(per)
    de = 2.0 * d * w[:, None] / n
    if d_eps_c is not None:
        d_eps_c.copy_(float(guidance) * de)
    if d_eps_u is not None:
        d_eps_u.copy_((1.0 - float(guidance)) * de)
