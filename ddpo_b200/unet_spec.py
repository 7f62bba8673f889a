"""Architecture spec + parameter manifest of the Stable-Diffusion U-Net the
reference drives through ``FlaxUNet2DConditionModel.apply`` (diffusers==0.12.1,
un-vendored; call sites ``ddpo/diffusers_patch/pipeline_flax_stable_diffusion.py:219-224``
and ``ddpo/training/policy_gradient.py:87-102``).

Parameter names and array layouts are the Flax checkpoint's: ``kernel`` is
``[in, out]`` for Dense and ``[kh, kw, in, out]`` (HWIO) for Conv, norms carry
``scale``/``bias``.  All parameters of one model live in ONE flat float32 buffer
(the optimizer, the gradient all-reduce and the checkpoint all see a single
array); the manifest maps names to (offset, shape) views.
"""
from dataclasses import dataclass
from typing import Dict, List, Tuple

import numpy as np
import torch


@dataclass(frozen=True)
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    # NB: in the Flax model ``attention_head_dim`` is the NUMBER OF HEADS per level
    attention_head_dim: Tuple[int, ...] = (5, 10, 20, 20)
    cross_attention_dim: int = 1024
    down_has_attn: Tuple[bool, ...] = (True, True, True, False)
    use_linear_projection: bool = True
    sample_size: int = 64
    norm_groups: int = 32
    ctx_len: int = 77

    @property
    def time_embed_dim(self):
        return self.block_out_channels[0] * 4


SD2_BASE = UNetConfig()
# the reference's own default checkpoint family (config/base.py:67); conv1x1 proj_in/out
SD1 = UNetConfig(attention_head_dim=(8, 8, 8, 8), cross_attention_dim=768, use_linear_projection=False)
# small configs for CPU-oracle-sized parity tests (same topology, d_head = 64)
TINY = UNetConfig(block_out_channels=(64, 128, 128, 128), attention_head_dim=(1, 2, 2, 2),
                  cross_attention_dim=64, sample_size=16, ctx_len=77)
SMALL = UNetConfig(block_out_channels=(128, 256, 256, 256), attention_head_dim=(2, 4, 4, 4),
                   cross_attention_dim=128, sample_size=32, ctx_len=77)


def _resnet(name, cin, cout, temb, out):
    out += [(f"{name}/norm1/scale", (cin,)), (f"{name}/norm1/bias", (cin,)),
            (f"{name}/conv1/kernel", (3, 3, cin, cout)), (f"{name}/conv1/bias", (cout,)),
            (f"{name}/time_emb_proj/kernel", (temb, cout)), (f"{name}/time_emb_proj/bias", (cout,)),
            (f"{name}/norm2/scale", (cout,)), (f"{name}/norm2/bias", (cout,)),
            (f"{name}/conv2/kernel", (3, 3, cout, cout)), (f"{name}/conv2/bias", (cout,))]
    if cin != cout:
        out += [(f"{name}/conv_shortcut/kernel", (1, 1, cin, cout)), (f"{name}/conv_shortcut/bias", (cout,))]


def _transformer(name, c, ctx, linear, out):
    out += [(f"{name}/norm/scale", (c,)), (f"{name}/norm/bias", (c,))]
    pk = (c, c) if linear else (1, 1, c, c)
    out += [(f"{name}/proj_in/kernel", pk), (f"{name}/proj_in/bias", (c,))]
    b = f"{name}/transformer_blocks_0"
    for i, kv in ((1, c), (2, ctx)):
        out += [(f"{b}/norm{i}/scale", (c,)), (f"{b}/norm{i}/bias", (c,)),
                (f"{b}/attn{i}/to_q/kernel", (c, c)), (f"{b}/attn{i}/to_k/kernel", (kv, c)),
                (f"{b}/attn{i}/to_v/kernel", (kv, c)),
                (f"{b}/attn{i}/to_out_0/kernel", (c, c)), (f"{b}/attn{i}/to_out_0/bias", (c,))]
    out += [(f"{b}/norm3/scale", (c,)), (f"{b}/norm3/bias", (c,)),
            (f"{b}/ff/net_0/proj/kernel", (c, 8 * c)), (f"{b}/ff/net_0/proj/bias", (8 * c,)),
            (f"{b}/ff/net_2/kernel", (4 * c, c)), (f"{b}/ff/net_2/bias", (c,))]
    out += [(f"{name}/proj_out/kernel", pk), (f"{name}/proj_out/bias", (c,))]


def param_manifest(cfg: UNetConfig) -> List[Tuple[str, Tuple[int, ...]]]:
    boc = cfg.block_out_channels
    te = cfg.time_embed_dim
    out: List[Tuple[str, Tuple[int, ...]]] = []
    out += [("conv_in/kernel", (3, 3, cfg.in_channels, boc[0])), ("conv_in/bias", (boc[0],)),
            ("time_embedding/linear_1/kernel", (boc[0], te)), ("time_embedding/linear_1/bias", (te,)),
            ("time_embedding/linear_2/kernel", (te, te)), ("time_embedding/linear_2/bias", (te,))]
    prev = boc[0]
    for i, c in enumerate(boc):
        for l in range(cfg.layers_per_block):
            _resnet(f"down_blocks_{i}/resnets_{l}", prev if l == 0 else c, c, te, out)
            if cfg.down_has_attn[i]:
                _transformer(f"down_blocks_{i}/attentions_{l}", c, cfg.cross_attention_dim,
                             cfg.use_linear_projection, out)
        if i < len(boc) - 1:
            out += [(f"down_blocks_{i}/downsamplers_0/conv/kernel", (3, 3, c, c)),
                    (f"down_blocks_{i}/downsamplers_0/conv/bias", (c,))]
        prev = c
    cm = boc[-1]
    _resnet("mid_block/resnets_0", cm, cm, te, out)
    _transformer("mid_block/attentions_0", cm, cfg.cross_attention_dim, cfg.use_linear_projection, out)
    _resnet("mid_block/resnets_1", cm, cm, te, out)
    rev = tuple(reversed(boc))
    has_attn = tuple(reversed(cfg.down_has_attn))
    prev_out = rev[0]
    for i, c in enumerate(rev):
        cin = rev[min(i + 1, len(rev) - 1)]
        n = cfg.layers_per_block + 1
        for l in range(n):
            skip = cin if l == n - 1 else c
            rin = prev_out if l == 0 else c
            _resnet(f"up_blocks_{i}/resnets_{l}", rin + skip, c, te, out)
            if has_attn[i]:
                _transformer(f"up_blocks_{i}/attentions_{l}", c, cfg.cross_attention_dim,
                             cfg.use_linear_projection, out)
        if i < len(rev) - 1:
            out += [(f"up_blocks_{i}/upsamplers_0/conv/kernel", (3, 3, c, c)),
                    (f"up_blocks_{i}/upsamplers_0/conv/bias", (c,))]
        prev_out = c
    out += [("conv_norm_out/scale", (boc[0],)), ("conv_norm_out/bias", (boc[0],)),
            ("conv_out/kernel", (3, 3, boc[0], cfg.out_channels)), ("conv_out/bias", (cfg.out_channels,))]
    return out


def param_offsets(cfg: UNetConfig, align: int = 64) -> Tuple[Dict[str, Tuple[int, Tuple[int, ...]]], int]:
    """name -> (offset in floats, shape); every tensor starts 256-byte aligned."""
    off = 0
    table = {}
    for name, shape in param_manifest(cfg):
        table[name] = (off, shape)
        n = int(np.prod(shape))
        off += (n + align - 1) // align * align
    return table, off


def num_params(cfg: UNetConfig) -> int:
    return sum(int(np.prod(s)) for _, s in param_manifest(cfg))


def init_flat_params(cfg: UNetConfig, seed: int = 0) -> torch.Tensor:
    """Random-init weights (synthetic; no checkpoints offline): fan-in-scaled normal
    kernels (Flax's lecun_normal scale), small random biases, norm scale 1+N(0,.1).
    Generated on the CPU so the oracle and the CUDA path see identical bytes."""
    table, total = param_offsets(cfg)
    g = torch.Generator(device="cpu").manual_seed(seed)
    flat = torch.zeros(total, dtype=torch.float32)
    for name, (off, shape) in table.items():
        n = int(np.prod(shape))
        leaf = name.rsplit("/", 1)[1]
        if leaf == "kernel":
            fan_in = int(np.prod(shape[:-1]))
            v = torch.randn(n, generator=g) * (1.0 / np.sqrt(fan_in))
        elif leaf == "scale":
            v = 1.0 + 0.1 * torch.randn(n, generator=g)
        else:
            v = 0.02 * torch.randn(n, generator=g)
        flat[off:off + n] = v
    return flat


def views(flat: torch.Tensor, cfg: UNetConfig) -> Dict[str, torch.Tensor]:
    table, _ = param_offsets(cfg)
    return {k: flat[o:o + int(np.prod(s))].view(*s) for k, (o, s) in table.items()}


# ------------------------------------------------------------------ LoRA adapters ----
LORA_RANKS = (4, 8, 16)
LORA_PROJECTIONS = ("to_q", "to_k", "to_v", "to_out_0")


def lora_manifest(cfg: UNetConfig, rank: int) -> List[Tuple[str, Tuple[int, ...], str]]:
    """(adapter name, shape, adapted kernel) of diffusers' LoRALinearLayer on the four projections of attn1 and attn2 in
    every transformer block: ``<attention>/<proj>/lora_down`` [in, rank] (down.weight^T) and ``.../lora_up`` [rank, out]
    (up.weight^T), in the U-Net's parameter order."""
    if rank not in LORA_RANKS:
        raise ValueError(f"lora_rank={rank!r}: must be one of {', '.join(map(str, LORA_RANKS))}")
    out = []
    for name, shape in param_manifest(cfg):
        parts = name.split("/")
        if len(parts) >= 3 and parts[-3] in ("attn1", "attn2") and parts[-2] in LORA_PROJECTIONS and parts[-1] == "kernel":
            base = name[: -len("/kernel")]
            k, n = shape
            out += [(base + "/lora_down", (k, rank), name), (base + "/lora_up", (rank, n), name)]
    return out


def lora_offsets(cfg: UNetConfig, rank: int, align: int = 64) -> Tuple[Dict[str, Tuple[int, Tuple[int, ...]]], int]:
    """adapter name -> (offset in floats, shape) in the flat fp32 adapter buffer; every tensor starts 256-byte aligned"""
    off = 0
    table = {}
    for name, shape, _ in lora_manifest(cfg, rank):
        table[name] = (off, shape)
        off += (int(np.prod(shape)) + align - 1) // align * align
    return table, off


def init_lora_params(cfg: UNetConfig, rank: int, seed: int = 0) -> torch.Tensor:
    """diffusers' LoRALinearLayer initialisation: down ~ N(0, (1/rank)^2), up = 0.  Drawn on the host from a seeded
    generator, so that every data-parallel rank builds the same adapters."""
    table, total = lora_offsets(cfg, rank)
    g = torch.Generator(device="cpu").manual_seed(seed)
    flat = torch.zeros(total, dtype=torch.float32)
    for name, (off, shape) in table.items():
        if name.endswith("/lora_down"):
            n = int(np.prod(shape))
            flat[off:off + n] = torch.randn(n, generator=g) * (1.0 / rank)
    return flat
