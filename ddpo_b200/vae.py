"""VAE decoder on the libddpo_b200 kernels -- what the reference reaches through
``pipeline.vae.apply({"params": vae_params}, latents / 0.18215, method=pipeline.vae.decode).sample`` followed by
``(images / 2 + 0.5).clip(0, 1).transpose(0, 2, 3, 1)`` (``pipeline/policy_gradient.py:174-182``,
``ddpo/training/diffusion.py:105-112``; 3P diffusers==0.12.1 ``vae_flax.py``: ``FlaxAutoencoderKL.decode`` =
``post_quant_conv`` -> ``FlaxDecoder``: conv_in, mid block (ResNet, single-head attention, ResNet), 4 up blocks of 3
ResNets (+ nearest-2x upsample conv on the first 3), GroupNorm(32, eps 1e-6) + swish, conv_out).

Parameter names / layouts are the Flax checkpoint's (``decoder/...``, ``post_quant_conv``; ``kernel`` = HWIO / [in, out]);
only the decoder half is held (the RWR path consumes stored posterior moments, it never encodes).

GPU design: the same building blocks as the U-Net -- bf16 implicit-GEMM convolutions with fp32 accumulators
(wgmma), fused bias / residual epilogues, one-pass GroupNorm+swish (statistics from the producing GEMM's epilogue) writing the bf16
GEMM operand, fp32 residual stream.  Pixel rows at the 256 / 512 px levels are wider than a 128-row tile: the igemm TMA producer walks them as
W/128 tiles per row.  The one attention layer has a single 512-wide head: scores are materialised per sample with two
GEMMs around a row-softmax kernel (Q K^T -> softmax -> P V, V^T produced directly by a GEMM with swapped operands);
at 0.4 % of a PPO sample's FLOPs a flash kernel for d = 512 is not worth its shared memory.  Images are decoded
``decode_batch`` at a time to bound the activation footprint (a 512x512x128 fp32 tensor is 134 MB per image).
"""
from dataclasses import dataclass
from typing import Dict, List, Tuple

import numpy as np
import torch

from . import ops
from .unet import Arena, _st

BF16, F32 = torch.bfloat16, torch.float32
GN_EPS = 1e-6          # 3P vae_flax.py: nn.GroupNorm(num_groups=32, epsilon=1e-6)
VAE_SCALING = 0.18215  # reference pipeline/policy_gradient.py:176


@dataclass(frozen=True)
class VAEConfig:
    latent_channels: int = 4
    out_channels: int = 3
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    sample_size: int = 64      # latent height / width


SD_VAE = VAEConfig()
# same topology at CPU-oracle size; 32x32 latents -> 256x256 images exercise the rows-wider-than-a-tile path
VAE_TINY = VAEConfig(block_out_channels=(64, 64, 128, 128), sample_size=32)
VAE_MICRO = VAEConfig(block_out_channels=(64, 64, 128, 128), sample_size=8)


def vae_config_for(pretrained_model):
    return {"tiny": VAE_MICRO, "small": VAE_TINY}.get(pretrained_model, SD_VAE)


def _resnet(name, cin, cout, out):
    out += [(f"{name}/norm1/scale", (cin,)), (f"{name}/norm1/bias", (cin,)),
            (f"{name}/conv1/kernel", (3, 3, cin, cout)), (f"{name}/conv1/bias", (cout,)),
            (f"{name}/norm2/scale", (cout,)), (f"{name}/norm2/bias", (cout,)),
            (f"{name}/conv2/kernel", (3, 3, cout, cout)), (f"{name}/conv2/bias", (cout,))]
    if cin != cout:
        out += [(f"{name}/conv_shortcut/kernel", (1, 1, cin, cout)), (f"{name}/conv_shortcut/bias", (cout,))]


def param_manifest(cfg: VAEConfig) -> List[Tuple[str, Tuple[int, ...]]]:
    lc = cfg.latent_channels
    rev = tuple(reversed(cfg.block_out_channels))
    out: List[Tuple[str, Tuple[int, ...]]] = [("post_quant_conv/kernel", (1, 1, lc, lc)), ("post_quant_conv/bias", (lc,)),
                                              ("decoder/conv_in/kernel", (3, 3, lc, rev[0])),
                                              ("decoder/conv_in/bias", (rev[0],))]
    c = rev[0]
    _resnet("decoder/mid_block/resnets_0", c, c, out)
    a = "decoder/mid_block/attentions_0"
    out += [(f"{a}/group_norm/scale", (c,)), (f"{a}/group_norm/bias", (c,))]
    for leaf in ("query", "key", "value", "proj_attn"):
        out += [(f"{a}/{leaf}/kernel", (c, c)), (f"{a}/{leaf}/bias", (c,))]
    _resnet("decoder/mid_block/resnets_1", c, c, out)
    prev = rev[0]
    for i, co in enumerate(rev):
        for l in range(cfg.layers_per_block + 1):
            _resnet(f"decoder/up_blocks_{i}/resnets_{l}", prev if l == 0 else co, co, out)
        if i < len(rev) - 1:
            out += [(f"decoder/up_blocks_{i}/upsamplers_0/conv/kernel", (3, 3, co, co)),
                    (f"decoder/up_blocks_{i}/upsamplers_0/conv/bias", (co,))]
        prev = co
    out += [("decoder/conv_norm_out/scale", (rev[-1],)), ("decoder/conv_norm_out/bias", (rev[-1],)),
            ("decoder/conv_out/kernel", (3, 3, rev[-1], cfg.out_channels)), ("decoder/conv_out/bias", (cfg.out_channels,))]
    return out


def encoder_param_manifest(cfg: VAEConfig) -> List[Tuple[str, Tuple[int, ...]]]:
    """``encoder/...`` + ``quant_conv`` of the Flax checkpoint (3P ``FlaxEncoder``): conv_in, per level two ResNets (+ a
    stride-2 ``downsamplers_0/conv`` on all but the last), mid block, conv_norm_out, conv_out -> 2 x latent channels."""
    lc, boc = cfg.latent_channels, cfg.block_out_channels
    out: List[Tuple[str, Tuple[int, ...]]] = [("encoder/conv_in/kernel", (3, 3, cfg.out_channels, boc[0])),
                                              ("encoder/conv_in/bias", (boc[0],))]
    prev = boc[0]
    for i, co in enumerate(boc):
        for l in range(cfg.layers_per_block):
            _resnet(f"encoder/down_blocks_{i}/resnets_{l}", prev if l == 0 else co, co, out)
        if i < len(boc) - 1:
            out += [(f"encoder/down_blocks_{i}/downsamplers_0/conv/kernel", (3, 3, co, co)),
                    (f"encoder/down_blocks_{i}/downsamplers_0/conv/bias", (co,))]
        prev = co
    c = boc[-1]
    _resnet("encoder/mid_block/resnets_0", c, c, out)
    a = "encoder/mid_block/attentions_0"
    out += [(f"{a}/group_norm/scale", (c,)), (f"{a}/group_norm/bias", (c,))]
    for leaf in ("query", "key", "value", "proj_attn"):
        out += [(f"{a}/{leaf}/kernel", (c, c)), (f"{a}/{leaf}/bias", (c,))]
    _resnet("encoder/mid_block/resnets_1", c, c, out)
    out += [("encoder/conv_norm_out/scale", (c,)), ("encoder/conv_norm_out/bias", (c,)),
            ("encoder/conv_out/kernel", (3, 3, c, 2 * lc)), ("encoder/conv_out/bias", (2 * lc,)),
            ("quant_conv/kernel", (1, 1, 2 * lc, 2 * lc)), ("quant_conv/bias", (2 * lc,))]
    return out


def param_offsets(cfg: VAEConfig, align: int = 64, part: str = "decoder"):
    off, table = 0, {}
    for name, shape in (param_manifest(cfg) if part == "decoder" else encoder_param_manifest(cfg)):
        table[name] = (off, shape)
        off += (int(np.prod(shape)) + align - 1) // align * align
    return table, off


def num_params(cfg: VAEConfig, part: str = "decoder") -> int:
    return sum(int(np.prod(s)) for _, s in (param_manifest(cfg) if part == "decoder" else encoder_param_manifest(cfg)))


def init_flat_params(cfg: VAEConfig, seed: int = 0, part: str = "decoder") -> torch.Tensor:
    """Random-init decoder (or encoder) weights (synthetic; no checkpoints offline): fan-in-scaled normal kernels, small
    biases, norm scale 1 + N(0, .1); generated on the CPU so the oracle and the CUDA path see identical bytes."""
    table, total = param_offsets(cfg, part=part)
    g = torch.Generator(device="cpu").manual_seed(seed)
    flat = torch.zeros(total, dtype=torch.float32)
    for name, (off, shape) in table.items():
        n = int(np.prod(shape))
        leaf = name.rsplit("/", 1)[1]
        if leaf == "kernel":
            v = torch.randn(n, generator=g) * (1.0 / np.sqrt(int(np.prod(shape[:-1]))))
        elif leaf == "scale":
            v = 1.0 + 0.1 * torch.randn(n, generator=g)
        else:
            v = 0.02 * torch.randn(n, generator=g)
        flat[off:off + n] = v
    return flat


def views(flat: torch.Tensor, cfg: VAEConfig, part: str = "decoder") -> Dict[str, torch.Tensor]:
    table, _ = param_offsets(cfg, part=part)
    return {k: flat[o:o + int(np.prod(s))].view(*s) for k, (o, s) in table.items()}


class _VAEHalf:
    """What the decoder and the encoder share: one flat fp32 parameter buffer in Flax layout, bf16 GEMM operands, an arena,
    and the two building blocks (ResNet without time embedding, single-head attention block)."""
    PART = "decoder"
    CUDA_CORE_LAYERS = ()   # layers that are not tensor-core shaped (K = 4 / 27 / 36, N = 3 / 8): fp32 CUDA-core kernels

    def __init__(self, cfg: VAEConfig = SD_VAE, flat_params: torch.Tensor = None, device="cuda", seed: int = 0,
                 decode_batch: int = 2):
        assert all(c % 64 == 0 for c in cfg.block_out_channels), "channel counts must be multiples of 64"
        assert cfg.latent_channels == 4 and cfg.out_channels == 3
        self.cfg = cfg
        self.device = torch.device(device)
        self.table, self.total = param_offsets(cfg, part=self.PART)
        if flat_params is None:
            flat_params = init_flat_params(cfg, seed, part=self.PART)
        assert flat_params.numel() == self.total
        self.params = flat_params.to(self.device, F32).contiguous()
        self.arena = Arena(self.device)
        self.decode_batch = int(decode_batch)
        self.w: Dict[str, torch.Tensor] = {}
        self.refresh_weights()

    def p(self, name):
        off, shape = self.table[name]
        return self.params[off:off + int(np.prod(shape))].view(*shape)

    def refresh_weights(self):
        """fp32 Flax params -> bf16 [N, K] GEMM operands (K = (tap, c_in))."""
        for name, (off, shape) in self.table.items():
            if not name.endswith("/kernel"):
                continue
            base = name[: -len("/kernel")]
            if base in self.CUDA_CORE_LAYERS:
                continue
            k, n = int(np.prod(shape[:-1])), int(shape[-1])
            if base not in self.w:
                self.w[base] = torch.empty(n, k, dtype=BF16, device=self.device)
            ops.prep_weight(self.p(name), self.w[base], k, n)

    # ------------------------------------------------------------------ blocks ----
    def _resnet(self, name, x, cin, cout, b, h, w):
        A = self.arena
        hw, m = h * w, b * h * w
        has_sc = (name + "/conv_shortcut/kernel") in self.table
        gws = A.alloc((ops.groupnorm_workspace_floats(b, hw, cin),), F32)
        a = A.alloc((m, cin), BF16)
        raw = A.alloc((m, cin), BF16) if has_sc else None
        ops.groupnorm_fwd(x, self.p(name + "/norm1/scale"), self.p(name + "/norm1/bias"), gws, b, hw, cin, silu=True,
                          y_bf16=a, raw_bf16=raw, eps=GN_EPS, stats0=_st(x))
        hbuf = A.alloc_with_gn_stats((m, cout), hw)   # the GEMM epilogue leaves the statistics norm2 needs
        ops.igemm(a0=a, wt=self.w[name + "/conv1"], n=cout, c0=cin, conv=(b, h, w), taps=9,
                  bias=self.p(name + "/conv1/bias"), out_f32=hbuf, gn_stats=_st(hbuf))
        A.release(a)
        A.release(gws)
        gws2 = A.alloc((ops.groupnorm_workspace_floats(b, hw, cout),), F32)
        a2 = A.alloc((m, cout), BF16)
        ops.groupnorm_fwd(hbuf, self.p(name + "/norm2/scale"), self.p(name + "/norm2/bias"), gws2, b, hw, cout,
                          silu=True, y_bf16=a2, eps=GN_EPS, stats0=_st(hbuf))
        A.release(hbuf)
        if has_sc:
            sc = A.alloc((m, cout), F32)
            ops.igemm(a0=raw, wt=self.w[name + "/conv_shortcut"], n=cout, c0=cin, conv=(b, h, w), taps=1,
                      bias=self.p(name + "/conv_shortcut/bias"), out_f32=sc)
            A.release(raw)
        else:
            sc = x
        out = A.alloc_with_gn_stats((m, cout), hw)
        ops.igemm(a0=a2, wt=self.w[name + "/conv2"], n=cout, c0=cout, conv=(b, h, w), taps=9,
                  bias=self.p(name + "/conv2/bias"), residual=sc, out_f32=out, gn_stats=_st(out))
        A.release(a2)
        A.release(gws2)
        if has_sc:
            A.release(sc)
        return out

    def _attention(self, name, x, c, b, h, w):
        """FlaxAttentionBlock, one head of width c: softmax((q s)(k s)^T) v with s = c^-1/4."""
        A = self.arena
        hw, m = h * w, b * h * w
        gws = A.alloc((ops.groupnorm_workspace_floats(b, hw, c),), F32)
        g = A.alloc((m, c), BF16)
        ops.groupnorm_fwd(x, self.p(name + "/group_norm/scale"), self.p(name + "/group_norm/bias"), gws, b, hw, c,
                          silu=False, y_bf16=g, eps=GN_EPS, stats0=_st(x))
        q = A.alloc((m, c), BF16)
        k = A.alloc((m, c), BF16)
        ops.igemm(a0=g, wt=self.w[name + "/query"], n=c, c0=c, m=m, bias=self.p(name + "/query/bias"), out_bf16=q)
        ops.igemm(a0=g, wt=self.w[name + "/key"], n=c, c0=c, m=m, bias=self.p(name + "/key/bias"), out_bf16=k)
        ao = A.alloc((m, c), BF16)
        vt = A.alloc((c, hw), BF16)
        scores = A.alloc((hw, hw), F32)
        probs = A.alloc((hw, hw), BF16)
        for s in range(b):
            rows = slice(s * hw, (s + 1) * hw)
            # V^T[c_out, pixel] = sum_k Wv[k, c_out] g[pixel, k]: the weight matrix is the row operand; the value
            # bias is added after P V (softmax rows sum to 1: P (V + 1 b^T) = P V + 1 b^T)
            ops.igemm(a0=self.w[name + "/value"], wt=g[rows], n=hw, c0=c, m=c, out_bf16=vt)
            ops.igemm(a0=q[rows], wt=k[rows], n=hw, c0=c, m=hw, out_f32=scores)
            ops.softmax_rows(scores, probs, 1.0 / float(np.sqrt(c)))
            ops.igemm(a0=probs, wt=vt, n=c, c0=hw, m=hw, bias=self.p(name + "/value/bias"), out_bf16=ao[rows])
        out = A.alloc_with_gn_stats((m, c), hw)
        ops.igemm(a0=ao, wt=self.w[name + "/proj_attn"], n=c, c0=c, m=m, bias=self.p(name + "/proj_attn/bias"),
                  residual=x, out_f32=out, gn_stats=_st(out))
        for t in (gws, g, q, k, ao, vt, scores, probs):
            A.release(t)
        return out



class VAEDecoder(_VAEHalf):
    PART = "decoder"
    CUDA_CORE_LAYERS = ("post_quant_conv", "decoder/conv_in", "decoder/conv_out")

    # ----------------------------------------------------------------- forward ----
    def _decode_chunk(self, latents, raw_out, img_out):
        cfg, A = self.cfg, self.arena
        b, lc, h, w = latents.shape
        rev = tuple(reversed(cfg.block_out_channels))
        z = A.alloc((b, lc, h, w), F32)
        ops.vae_post_quant(latents, self.p("post_quant_conv/kernel"), self.p("post_quant_conv/bias"), z,
                           scaling=VAE_SCALING)
        c = rev[0]
        x = A.alloc_with_gn_stats((b * h * w, c), h * w)
        ops.conv_in(z, self.p("decoder/conv_in/kernel"), self.p("decoder/conv_in/bias"), x, b, lc, h, w, c, gn_stats=_st(x))
        A.release(z)
        for name, kind in (("decoder/mid_block/resnets_0", "r"), ("decoder/mid_block/attentions_0", "a"),
                           ("decoder/mid_block/resnets_1", "r")):
            y = self._resnet(name, x, c, c, b, h, w) if kind == "r" else self._attention(name, x, c, b, h, w)
            A.release(x)
            x = y
        prev = c
        for i, co in enumerate(rev):
            for l in range(cfg.layers_per_block + 1):
                y = self._resnet(f"decoder/up_blocks_{i}/resnets_{l}", x, prev if l == 0 else co, co, b, h, w)
                A.release(x)
                x = y
            if i < len(rev) - 1:
                name = f"decoder/up_blocks_{i}/upsamplers_0"
                up = A.alloc((b * 4 * h * w, co), BF16)
                ops.upsample2x_bf16(x, up, b, h, w, co)      # jax.image.resize(nearest): out[i] = in[i // 2]
                A.release(x)
                h, w = 2 * h, 2 * w
                x = A.alloc_with_gn_stats((b * h * w, co), h * w)
                ops.igemm(a0=up, wt=self.w[name + "/conv"], n=co, c0=co, conv=(b, h, w), taps=9,
                          bias=self.p(name + "/conv/bias"), out_f32=x, gn_stats=_st(x))
                A.release(up)
            prev = co
        c0 = rev[-1]
        gws = A.alloc((ops.groupnorm_workspace_floats(b, h * w, c0),), F32)
        yf = A.alloc((b * h * w, c0), F32)
        ops.groupnorm_fwd(x, self.p("decoder/conv_norm_out/scale"), self.p("decoder/conv_norm_out/bias"), gws, b, h * w,
                          c0, silu=True, y_f32=yf, eps=GN_EPS, stats0=_st(x))
        ops.vae_conv_out(yf, self.p("decoder/conv_out/kernel"), self.p("decoder/conv_out/bias"), b, h, w, c0,
                         raw_nchw=raw_out, img_nhwc=img_out)
        for t in (x, gws, yf):
            A.release(t)

    @torch.no_grad()
    def decode(self, latents: torch.Tensor, want_raw: bool = False, want_images: bool = True):
        """latents fp32 NCHW [B,4,h,w] (as sampled, i.e. still multiplied by 0.18215) ->
        ``images`` fp32 NHWC [B,8h,8w,3] in [0,1] and/or ``raw`` fp32 NCHW [B,3,8h,8w] (the decoder's ``.sample``)."""
        latents = latents.to(self.device, F32).contiguous()
        B, _, h, w = latents.shape
        up = 2 ** (len(self.cfg.block_out_channels) - 1)
        H, W = h * up, w * up
        raw = torch.empty(B, 3, H, W, device=self.device) if want_raw else None
        img = torch.empty(B, H, W, 3, device=self.device) if want_images else None
        for s in range(0, B, self.decode_batch):
            e = min(B, s + self.decode_batch)
            self._decode_chunk(latents[s:e], None if raw is None else raw[s:e], None if img is None else img[s:e])
        return (img, raw) if want_raw and want_images else (raw if want_raw else img)

    def decode_to_images(self, latents):
        return self.decode(latents, want_raw=False, want_images=True)

    __call__ = decode_to_images


class VAEEncoder(_VAEHalf):
    """VAE encoder on the same kernels -- what the reference's ``vae_fn`` computes for the RWR data path
    (``ddpo/training/callbacks.py:37-57``: ``(images - 0.5) / 0.5`` -> 3P ``FlaxAutoencoderKL.encode`` ->
    ``concatenate([latent_dist.mean, latent_dist.logvar], -1)``): conv_in, per level two ResNets and a stride-2 down-sample
    whose Flax padding ((0,1),(0,1)) + VALID is the implicit GEMM's ``no_low_pad`` tap geometry (reads past the high edge
    are TMA zero fill), mid block, GroupNorm + swish, then the fp32 head (conv_out to 8 channels, ``quant_conv`` 1x1, logvar
    clip to [-30, 20]).  Parameter names / layouts are the Flax checkpoint's (``encoder/...``, ``quant_conv``)."""
    PART = "encoder"
    CUDA_CORE_LAYERS = ("encoder/conv_in", "encoder/conv_out", "quant_conv")

    def _encode_chunk(self, images, moments_out):
        cfg, A = self.cfg, self.arena
        b, H, W, _ = images.shape
        boc = cfg.block_out_channels
        xin = A.alloc((b, 3, H, W), F32)
        ops.vae_image_to_nchw(images, xin)
        c, h, w = boc[0], H, W
        x = A.alloc_with_gn_stats((b * h * w, c), h * w)
        ops.conv_in(xin, self.p("encoder/conv_in/kernel"), self.p("encoder/conv_in/bias"), x, b, 3, h, w, c, gn_stats=_st(x))
        A.release(xin)
        prev = c
        for i, co in enumerate(boc):
            for l in range(cfg.layers_per_block):
                y = self._resnet(f"encoder/down_blocks_{i}/resnets_{l}", x, prev if l == 0 else co, co, b, h, w)
                A.release(x)
                x = y
            if i < len(boc) - 1:
                name = f"encoder/down_blocks_{i}/downsamplers_0"
                xb = A.alloc((b * h * w, co), BF16)
                ops.cast_bf16(x, xb)
                A.release(x)
                h, w = h // 2, w // 2
                x = A.alloc_with_gn_stats((b * h * w, co), h * w)
                ops.igemm(a0=xb, wt=self.w[name + "/conv"], n=co, c0=co, conv=(b, h, w), taps=9, stride=2, no_low_pad=True,
                          bias=self.p(name + "/conv/bias"), out_f32=x, gn_stats=_st(x))
                A.release(xb)
            prev = co
        c = boc[-1]
        for name, kind in (("encoder/mid_block/resnets_0", "r"), ("encoder/mid_block/attentions_0", "a"),
                           ("encoder/mid_block/resnets_1", "r")):
            y = self._resnet(name, x, c, c, b, h, w) if kind == "r" else self._attention(name, x, c, b, h, w)
            A.release(x)
            x = y
        gws = A.alloc((ops.groupnorm_workspace_floats(b, h * w, c),), F32)
        yf = A.alloc((b * h * w, c), F32)
        ops.groupnorm_fwd(x, self.p("encoder/conv_norm_out/scale"), self.p("encoder/conv_norm_out/bias"), gws, b, h * w, c,
                          silu=True, y_f32=yf, eps=GN_EPS, stats0=_st(x))
        ops.vae_encoder_head(yf, self.p("encoder/conv_out/kernel"), self.p("encoder/conv_out/bias"),
                             self.p("quant_conv/kernel"), self.p("quant_conv/bias"), moments_out, b, h, w, c)
        for t in (x, gws, yf):
            A.release(t)

    @torch.no_grad()
    def encode(self, images: torch.Tensor):
        """images fp32 NHWC [B, H, W, 3] in [0, 1] -> posterior moments fp32 NHWC [B, H/8, W/8, 8] (mean | logvar)."""
        images = torch.as_tensor(images).to(self.device, F32).contiguous()
        B, H, W, _ = images.shape
        down = 2 ** (len(self.cfg.block_out_channels) - 1)
        out = torch.empty(B, H // down, W // down, 2 * self.cfg.latent_channels, device=self.device)
        for s in range(0, B, self.decode_batch):
            e = min(B, s + self.decode_batch)
            self._encode_chunk(images[s:e], out[s:e])
        return out

    __call__ = encode
