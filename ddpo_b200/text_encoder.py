"""CLIP text encoder on the libddpo_b200 kernels -- what the reference calls as
``pipeline.text_encoder(input_ids, params=params["text_encoder"])[0]`` (``pipeline/policy_gradient.py:185-187`` on the
host CPU "to save memory"; ``ddpo/training/diffusion.py:45-51,62-68`` inside the RWR step; 3P transformers==4.28.1
``FlaxCLIPTextModel``): token + position embeddings, N pre-LayerNorm transformer layers with CAUSAL self-attention
(heads of width 64, q scaled by d^-1/2) and a two-layer MLP (``gelu`` for the OpenCLIP ViT-H text tower of SD2,
``quick_gelu`` for the CLIP-L tower of SD1), final LayerNorm; returns the last hidden state ``[B, 77, D]`` fp32.

Parameter names / layouts are the Flax checkpoint's (``text_model/encoder/layers/<i>/self_attn/q_proj/kernel`` is
``[in, out]`` ...).  SD2 keeps 23 of ViT-H's 24 layers (the penultimate-layer conditioning is baked into the config).

GPU design: 77-token sequences are tiny (4.5 GFLOP per prompt for SD2) -- the win is not the FLOPs but removing the
host-CPU stall and the H2D of the embeddings from every sample batch: q/k/v are one fused GEMM, attention is the U-Net's
wgmma flash kernel with the causal bound added to its key mask, bias / residual ride in the GEMM epilogues."""
from dataclasses import dataclass
from typing import Dict, List, Tuple

import numpy as np
import torch

from . import ops
from .unet import Arena

BF16, F32 = torch.bfloat16, torch.float32


@dataclass(frozen=True)
class CLIPTextConfig:
    vocab_size: int = 49408
    hidden_size: int = 1024
    intermediate_size: int = 4096
    num_hidden_layers: int = 23
    num_attention_heads: int = 16
    max_position_embeddings: int = 77
    hidden_act: str = "gelu"
    layer_norm_eps: float = 1e-5


SD2_TEXT = CLIPTextConfig()
SD1_TEXT = CLIPTextConfig(hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                          hidden_act="quick_gelu")
CLIP_B32_TEXT = CLIPTextConfig(hidden_size=512, intermediate_size=2048, num_hidden_layers=12, num_attention_heads=8,
                               hidden_act="quick_gelu")     # openai/clip-vit-base-patch32 (the consistency reward)
TEXT_TINY = CLIPTextConfig(vocab_size=1000, hidden_size=128, intermediate_size=512, num_hidden_layers=2,
                           num_attention_heads=2)
TEXT_TINY_QUICK = CLIPTextConfig(vocab_size=1000, hidden_size=192, intermediate_size=256, num_hidden_layers=1,
                                 num_attention_heads=3, hidden_act="quick_gelu")


def text_config_for(pretrained_model):
    """the text tower that conditions the U-Net of ``pretrained_model`` (hidden size == cross_attention_dim)"""
    from .utils.serialization import MODEL_CONFIGS
    if MODEL_CONFIGS.get(pretrained_model) == "SD1":
        return SD1_TEXT
    return {"tiny": CLIPTextConfig(vocab_size=49408, hidden_size=64, intermediate_size=256, num_hidden_layers=2,
                                   num_attention_heads=1),
            "small": CLIPTextConfig(vocab_size=49408, hidden_size=128, intermediate_size=512, num_hidden_layers=2,
                                    num_attention_heads=2)}.get(pretrained_model, SD2_TEXT)


def param_manifest(cfg: CLIPTextConfig) -> List[Tuple[str, Tuple[int, ...]]]:
    D, I = cfg.hidden_size, cfg.intermediate_size
    out = [("text_model/embeddings/token_embedding/embedding", (cfg.vocab_size, D)),
           ("text_model/embeddings/position_embedding/embedding", (cfg.max_position_embeddings, D))]
    for i in range(cfg.num_hidden_layers):
        b = f"text_model/encoder/layers/{i}"
        out += [(f"{b}/layer_norm1/scale", (D,)), (f"{b}/layer_norm1/bias", (D,))]
        for p in ("q_proj", "k_proj", "v_proj", "out_proj"):
            out += [(f"{b}/self_attn/{p}/kernel", (D, D)), (f"{b}/self_attn/{p}/bias", (D,))]
        out += [(f"{b}/layer_norm2/scale", (D,)), (f"{b}/layer_norm2/bias", (D,)),
                (f"{b}/mlp/fc1/kernel", (D, I)), (f"{b}/mlp/fc1/bias", (I,)),
                (f"{b}/mlp/fc2/kernel", (I, D)), (f"{b}/mlp/fc2/bias", (D,))]
    out += [("text_model/final_layer_norm/scale", (D,)), ("text_model/final_layer_norm/bias", (D,))]
    return out


def param_offsets(cfg: CLIPTextConfig, align: int = 64):
    off, table = 0, {}
    for name, shape in param_manifest(cfg):
        table[name] = (off, shape)
        off += (int(np.prod(shape)) + align - 1) // align * align
    return table, off


def num_params(cfg: CLIPTextConfig) -> int:
    return sum(int(np.prod(s)) for _, s in param_manifest(cfg))


def init_flat_params(cfg: CLIPTextConfig, seed: int = 0) -> torch.Tensor:
    """Random-init weights (synthetic: no checkpoints offline), generated on the CPU for oracle / CUDA byte identity."""
    table, total = param_offsets(cfg)
    g = torch.Generator(device="cpu").manual_seed(seed)
    flat = torch.zeros(total, dtype=torch.float32)
    for name, (off, shape) in table.items():
        n = int(np.prod(shape))
        leaf = name.rsplit("/", 1)[1]
        if leaf == "kernel":
            v = torch.randn(n, generator=g) / np.sqrt(shape[0])
        elif leaf == "embedding":
            v = 0.5 * torch.randn(n, generator=g)
        elif leaf == "scale":
            v = 1.0 + 0.1 * torch.randn(n, generator=g)
        else:
            v = 0.02 * torch.randn(n, generator=g)
        flat[off:off + n] = v
    return flat


def views(flat: torch.Tensor, cfg: CLIPTextConfig) -> Dict[str, torch.Tensor]:
    table, _ = param_offsets(cfg)
    return {k: flat[o:o + int(np.prod(s))].view(*s) for k, (o, s) in table.items()}


class CLIPTextEncoder:
    """``encoder(input_ids, params=None, train=False) -> (last_hidden_state,)`` like ``FlaxCLIPTextModel``."""

    def __init__(self, cfg: CLIPTextConfig = SD2_TEXT, flat_params: torch.Tensor = None, device="cuda", seed: int = 0):
        assert cfg.hidden_size % 64 == 0 and cfg.hidden_size // cfg.num_attention_heads == 64, "head width must be 64"
        assert cfg.intermediate_size % 64 == 0
        self.cfg = cfg
        self.device = torch.device(device)
        self.table, self.total = param_offsets(cfg)
        if flat_params is None:
            flat_params = init_flat_params(cfg, seed)
        assert flat_params.numel() == self.total
        self.params = flat_params.to(self.device, F32).contiguous()
        self.arena = Arena(self.device)
        self.w: Dict[str, torch.Tensor] = {}
        self.qkv_bias: Dict[str, torch.Tensor] = {}
        self.refresh_weights()

    def p(self, name):
        off, shape = self.table[name]
        return self.params[off:off + int(np.prod(shape))].view(*shape)

    def refresh_weights(self):
        """fp32 Flax params -> bf16 [N, K] GEMM operands; q/k/v fused into one [3D, D] operand (+ fused bias)."""
        D, I = self.cfg.hidden_size, self.cfg.intermediate_size
        for i in range(self.cfg.num_hidden_layers):
            b = f"text_model/encoder/layers/{i}"
            key = b + "/self_attn/qkv"
            if key not in self.w:
                self.w[key] = torch.empty(3 * D, D, dtype=BF16, device=self.device)
                self.qkv_bias[key] = torch.empty(3 * D, dtype=F32, device=self.device)
            for j, pn in enumerate(("q_proj", "k_proj", "v_proj")):
                ops.prep_weight(self.p(f"{b}/self_attn/{pn}/kernel"), self.w[key], D, D, row_offset=j * D)
                self.qkv_bias[key][j * D:(j + 1) * D].copy_(self.p(f"{b}/self_attn/{pn}/bias"))
            for name, k, n in ((b + "/self_attn/out_proj", D, D), (b + "/mlp/fc1", D, I), (b + "/mlp/fc2", I, D)):
                if name not in self.w:
                    self.w[name] = torch.empty(n, k, dtype=BF16, device=self.device)
                ops.prep_weight(self.p(name + "/kernel"), self.w[name], k, n)

    @torch.no_grad()
    def encode(self, input_ids) -> torch.Tensor:
        cfg, A = self.cfg, self.arena
        ids = torch.as_tensor(np.asarray(input_ids)) if not torch.is_tensor(input_ids) else input_ids
        B, L = ids.shape
        if L > cfg.max_position_embeddings:
            raise ValueError(f"sequence length {L} exceeds max_position_embeddings {cfg.max_position_embeddings}")
        D, I, H = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads
        m = B * L
        ids_dev = ids.to(self.device, torch.int32).reshape(m).contiguous()
        x = A.alloc((m, D), F32)
        ops.embed_tokens(ids_dev, self.p("text_model/embeddings/token_embedding/embedding"),
                         self.p("text_model/embeddings/position_embedding/embedding"), x, L)
        for i in range(cfg.num_hidden_layers):
            b = f"text_model/encoder/layers/{i}"
            ln = A.alloc((m, D), BF16)
            ops.layernorm_fwd(x, self.p(b + "/layer_norm1/scale"), self.p(b + "/layer_norm1/bias"), ln, m, D)
            qkv = A.alloc((m, 3 * D), BF16)
            ops.igemm(a0=ln, wt=self.w[b + "/self_attn/qkv"], n=3 * D, c0=D, m=m, bias=self.qkv_bias[b + "/self_attn/qkv"],
                      out_bf16=qkv)
            ao = A.alloc((m, D), BF16)
            ops.attention_fwd(qkv, qkv[:, D:], qkv[:, 2 * D:], ao, B, H, L, L, 3 * D, 3 * D, 3 * D, D, causal=True)
            h1 = A.alloc((m, D), F32)
            ops.igemm(a0=ao, wt=self.w[b + "/self_attn/out_proj"], n=D, c0=D, m=m,
                      bias=self.p(b + "/self_attn/out_proj/bias"), residual=x, out_f32=h1)
            ops.layernorm_fwd(h1, self.p(b + "/layer_norm2/scale"), self.p(b + "/layer_norm2/bias"), ln, m, D)
            f1 = A.alloc((m, I), F32)
            ops.igemm(a0=ln, wt=self.w[b + "/mlp/fc1"], n=I, c0=D, m=m, bias=self.p(b + "/mlp/fc1/bias"), out_f32=f1)
            fa = A.alloc((m, I), BF16)
            ops.act_bf16(f1, fa, cfg.hidden_act)
            x2 = A.alloc((m, D), F32)
            ops.igemm(a0=fa, wt=self.w[b + "/mlp/fc2"], n=D, c0=I, m=m, bias=self.p(b + "/mlp/fc2/bias"), residual=h1,
                      out_f32=x2)
            for t in (ln, qkv, ao, h1, f1, fa, x):
                A.release(t)
            x = x2
        out = torch.empty(B, L, D, dtype=F32, device=self.device)
        ops.layernorm_f32(x, self.p("text_model/final_layer_norm/scale"), self.p("text_model/final_layer_norm/bias"),
                          out.view(m, D), m, D, eps=cfg.layer_norm_eps)
        A.release(x)
        return out

    def __call__(self, input_ids, params=None, train=False):
        return (self.encode(input_ids),)
