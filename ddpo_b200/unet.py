"""Host-side assembly of the Stable-Diffusion U-Net on the libddpo_b200 kernels.

Mirrors what the reference reaches through ``pipeline.unet.apply({"params": p}, latents,
timesteps, encoder_hidden_states).sample`` (3P diffusers==0.12.1 FlaxUNet2DConditionModel;
reference call sites ``ddpo/diffusers_patch/pipeline_flax_stable_diffusion.py:219-224`` and
``ddpo/training/policy_gradient.py:87-102``), with the Flax semantics listed in
``ddpo_b200/unet_spec.py``.  This file only sequences kernel launches and owns buffers;
all arithmetic happens in the CUDA library.

Data flow design:
  * the residual stream is fp32 NHWC; every GEMM/conv A operand is the bf16 output of the
    preceding norm kernel; accumulation is fp32 (wgmma register accumulators); bias / time-embedding / residual /
    GEGLU are fused in GEMM epilogues;
  * U-Net skip concatenations are never materialised (two-source norm + two-source conv);
  * cross-attention K/V projections depend only on the text context and are computed once per
    prompt batch (``prepare_context``), not once per denoising step;
  * buffers come from a deterministic free-list arena so a whole step can be captured in a
    CUDA graph.
"""
from typing import Dict, List, Optional

import numpy as np
import torch

from . import ops
from .ops import ATTENTION_HEAD_DIMS
from .unet_spec import UNetConfig, init_lora_params, lora_manifest, lora_offsets, param_offsets

BF16 = torch.bfloat16
F32 = torch.float32


def _st(t):
    """slab statistics the producing GEMM left for tensor ``t`` (None: the GroupNorm computes them itself)"""
    return getattr(t, "_gn_stats", None) if t is not None else None


class Arena:
    """Deterministic free-list allocator (persistent torch tensors, reused by byte size)."""

    def __init__(self, device):
        self.device = device
        self.free: Dict[int, List[torch.Tensor]] = {}
        self.total_bytes = 0

    def alloc(self, shape, dtype):
        n = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
        n = (n + 255) // 256 * 256
        lst = self.free.get(n)
        if lst:
            raw = lst.pop()
        else:
            raw = torch.empty(n, dtype=torch.uint8, device=self.device)
            self.total_bytes += n
        t = raw[: int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()].view(dtype).view(*shape)
        t._ddpo_raw = raw
        return t

    def alloc_with_gn_stats(self, shape, hw):
        """fp32 [rows, channels] GEMM output plus, when a sample's pixels fill whole 32-row slabs, the slab-statistics
        buffer the GEMM epilogue writes for the GroupNorm that will consume it (``ops.igemm(gn_stats=...)``).  The
        statistics travel with the tensor (``t._gn_stats``) and are released with it."""
        t = self.alloc(shape, F32)
        t._gn_stats = self.alloc(ops.gn_stats_shape(shape[0], shape[1]), F32) if hw % 32 == 0 else None
        return t

    def release(self, t):
        if t is None:
            return
        st = getattr(t, "_gn_stats", None)
        if st is not None:
            t._gn_stats = None
            self.release(st)
        raw = getattr(t, "_ddpo_raw", None)
        if raw is not None:
            self.free.setdefault(raw.numel(), []).append(raw)
            t._ddpo_raw = None


def _head_dim_kw(c, heads):
    """the ``head_dim`` keyword of the ops' attention calls: omitted at 64, the ops' default, so that an ops module without
    the keyword (the torch-CPU emulation the host-assembly dry runs use, tests/_cpu_ops_emulator.py) runs the SD2 family"""
    d = c // heads
    return {} if d == 64 else {"head_dim": d}


class UNet:
    def __init__(self, cfg: UNetConfig, flat_params: torch.Tensor, device="cuda"):
        assert all(c % 64 == 0 for c in cfg.block_out_channels), "channel counts must be multiples of 64"
        for c, h in zip(cfg.block_out_channels, cfg.attention_head_dim):
            assert c % h == 0 and c // h in ATTENTION_HEAD_DIMS, \
                f"{c} channels over {h} heads: the attention kernels take head dims {ATTENTION_HEAD_DIMS} " \
                "(SD2: 64, SD1.x: 40, 80, 160)"
        assert cfg.cross_attention_dim % 64 == 0
        self.cfg = cfg
        self.device = torch.device(device)
        self.table, self.total = param_offsets(cfg)
        assert flat_params.numel() == self.total
        self.params = flat_params.to(self.device, F32).contiguous()
        self.arena = Arena(self.device)
        self.w: Dict[str, torch.Tensor] = {}       # bf16 forward GEMM operands
        self.aux: Dict[str, torch.Tensor] = {}     # permuted biases etc.
        self.ctx_kv: Optional[Dict[str, torch.Tensor]] = None
        self._ctx_cache: Dict[tuple, dict] = {}     # context shape -> persistent bf16 context + K/V buffers
        self.ctx_batch = 0
        self._layers = self._enumerate_layers()
        self.wd: Dict[str, torch.Tensor] = {}      # bf16 backward (dgrad) GEMM operands, built on demand
        self.grads: Optional[torch.Tensor] = None  # flat fp32 gradient accumulator (same layout as params)
        self.train_mode = False
        # all ResNet time-embedding projections of a pass in ONE launch (ops.dense_small_grouped): bit-identical to the 22
        # separate dense_small launches (tests/test_gpu_kernels.py), each of which runs only 10-40 CTAs.
        self._temb_names = [n[: -len("/time_emb_proj/kernel")] for n in self.table if n.endswith("/time_emb_proj/kernel")]
        self._temb_tables: Dict[int, tuple] = {}
        self._tproj_views: Optional[Dict[str, torch.Tensor]] = None
        # LoRA mode (enable_lora): the U-Net is frozen and only the adapters of the attention projections train
        self.lora_rank = 0
        self.lora_params: Optional[torch.Tensor] = None   # flat fp32 adapters (lora_table layout)
        self.lora_grads: Optional[torch.Tensor] = None
        self.lora_table: Dict[str, tuple] = {}
        self.refresh_weights()

    # ------------------------------------------------------------------ params ----
    def p(self, name):
        off, shape = self.table[name]
        return self.params[off:off + int(np.prod(shape))].view(*shape)

    def _enumerate_layers(self):
        """(kind, name, ...) for every tensor-core GEMM weight."""
        cfg = self.cfg
        out = []
        for name, shape in ((k, v[1]) for k, v in self.table.items()):
            if not name.endswith("/kernel"):
                continue
            base = name[: -len("/kernel")]
            if base in ("conv_in", "conv_out") or base.startswith("time_embedding") or base.endswith("time_emb_proj"):
                continue
            out.append((base, shape))
        return out

    def _lora_views(self, base):
        """(down, up) adapter views of an adapted layer, or None"""
        if base + "/lora_down" not in self.lora_table:
            return None
        return self.lp(base + "/lora_down"), self.lp(base + "/lora_up")

    def refresh_weights(self):
        """fp32 Flax params -> bf16 [N, K] GEMM operands (run after every optimizer step).  In LoRA mode the adapted
        layers' operands are bf16(W + D U) (ops.lora_merge), and once built only those are re-merged: nothing else
        changes."""
        adapted_only = self.lora_rank > 0 and getattr(self, "_frozen_ready", False)
        for base, shape in self._layers:
            leaf = base.rsplit("/", 1)[1]
            lora = self._lora_views(base)
            if adapted_only and lora is None:
                continue
            src = self.p(base + "/kernel")
            k = int(np.prod(shape[:-1]))
            n = int(shape[-1])

            def prep(dst, row_offset=0):
                if lora is None:
                    ops.prep_weight(src, dst, k, n, row_offset=row_offset)
                else:
                    ops.lora_merge(src, lora[0], lora[1], k, n, self.lora_rank, fwd=dst, ldk=k, row_offset=row_offset)
            if leaf in ("to_q", "to_k", "to_v"):
                attn = base.rsplit("/", 1)[0]
                is_self = attn.endswith("attn1")
                if is_self:
                    key = attn + "/qkv"
                    if key not in self.w:
                        self.w[key] = torch.empty(3 * n, k, dtype=BF16, device=self.device)
                    prep(self.w[key], row_offset={"to_q": 0, "to_k": n, "to_v": 2 * n}[leaf])
                elif leaf == "to_q":
                    key = attn + "/q"
                    if key not in self.w:
                        self.w[key] = torch.empty(n, k, dtype=BF16, device=self.device)
                    prep(self.w[key])
                else:
                    key = attn + "/kv"
                    if key not in self.w:
                        self.w[key] = torch.empty(2 * n, k, dtype=BF16, device=self.device)
                    prep(self.w[key], row_offset=0 if leaf == "to_k" else n)
                continue
            if lora is not None:                   # to_out_0
                if base not in self.w:
                    self.w[base] = torch.empty(n, k, dtype=BF16, device=self.device)
                prep(self.w[base])
                continue
            if base not in self.w:
                self.w[base] = torch.empty(n, k, dtype=BF16, device=self.device)
            if base.endswith("ff/net_0/proj"):
                ops.prep_weight(src, self.w[base], k, n, geglu_bn=256)
                if base not in self.aux:
                    self.aux[base] = torch.empty(n, dtype=F32, device=self.device)
                ops.permute_geglu_bias(self.p(base + "/bias"), self.aux[base], n, 256)
            else:
                ops.prep_weight(src, self.w[base], k, n)
        if self.train_mode:
            self._refresh_dgrad_weights(adapted_only)
        if self.lora_rank > 0 and self.train_mode:
            self._frozen_ready = True

    def enable_training(self):
        """Allocates the gradient accumulator (full fine-tuning only: in LoRA mode the adapters' gradient buffer is
        ``lora_grads``) and the dgrad-layout bf16 weights."""
        if self.grads is None and self.lora_rank == 0:
            self.grads = torch.zeros_like(self.params)
        self.train_mode = True
        self._refresh_dgrad_weights(False)
        if self.lora_rank > 0:
            self._frozen_ready = True

    def enable_lora(self, rank: int, seed: int = 0):
        """LoRA mode: rank-``rank`` adapters (diffusers' LoRALinearLayer, scale 1) on to_q / to_k / to_v / to_out_0 of
        both attentions of every transformer block, the rest of the U-Net frozen.  Builds the adapter table, the flat
        fp32 adapters (down ~ N(0, 1/rank^2), up = 0, from a seeded host generator) and their gradient buffer; the
        U-Net's own gradient buffer is never allocated.  Call before ``enable_training``."""
        assert self.grads is None, "enable_lora() on a U-Net that already trains all of its parameters"
        self.lora_table, total = lora_offsets(self.cfg, rank)
        self.lora_rank = int(rank)
        self.lora_params = init_lora_params(self.cfg, rank, seed).to(self.device)
        self.lora_grads = torch.zeros(total, dtype=F32, device=self.device)
        # where the kernels that always produce a parameter gradient (norm backwards, conv_out) put it in LoRA mode;
        # kernel / scale and bias get separate halves
        self._discard = torch.zeros(2, 16384, dtype=F32, device=self.device)
        self._frozen_ready = False
        self.refresh_weights()
        return self

    def lp(self, name):
        off, shape = self.lora_table[name]
        return self.lora_params[off:off + int(np.prod(shape))].view(*shape)

    def lg(self, name):
        off, shape = self.lora_table[name]
        return self.lora_grads[off:off + int(np.prod(shape))].view(*shape)

    def merged_params(self) -> torch.Tensor:
        """The flat fp32 parameters, in host memory, with every adapted kernel replaced by W + D U (the U-Net the
        adapters define; what a checkpoint of a LoRA run holds).  Without adapters: a host copy of ``params``.  The
        kernels are merged one at a time through a small device buffer, so that saving a checkpoint does not hold a
        second copy of the U-Net on the device."""
        out = self.params.cpu().clone() if self.params.is_cuda else self.params.clone()
        scratch = None
        for _, _, kernel in lora_manifest(self.cfg, self.lora_rank)[::2] if self.lora_rank else ():
            base = kernel[: -len("/kernel")]
            off, (k, n) = self.table[kernel]
            if scratch is None or scratch.numel() < k * n:
                scratch = torch.empty(k * n, dtype=F32, device=self.device)
            down, up = self._lora_views(base)
            merged = scratch[:k * n].view(k, n)
            ops.lora_merge(self.p(base + "/kernel"), down, up, k, n, self.lora_rank, merged=merged)
            out[off:off + k * n].copy_(merged.reshape(-1))
        return out

    def _refresh_dgrad_weights(self, adapted_only=False):
        for base, shape in self._layers:
            leaf = base.rsplit("/", 1)[1]
            if leaf in ("to_k", "to_v") and "/attn2/" in base:
                continue  # the text context receives no gradient
            lora = self._lora_views(base)
            if adapted_only and lora is None:
                continue
            cin, n = int(shape[-2]), int(shape[-1])

            def prep(dst, ld_dst=0, col_offset=0):
                if lora is None:
                    ops.prep_weight_dgrad(self.p(base + "/kernel"), dst, 1, cin, n, ld_dst=ld_dst, col_offset=col_offset)
                else:
                    ops.lora_merge(self.p(base + "/kernel"), lora[0], lora[1], cin, n, self.lora_rank, dgrad=dst,
                                   ld_dst=ld_dst, col_offset=col_offset)
            if leaf in ("to_q", "to_k", "to_v") and "/attn1/" in base:
                # the input gradient of self-attention is ONE GEMM over K = 3C: d_ln = [dq | dk | dv] [Wq | Wk | Wv]^T
                key = base.rsplit("/", 1)[0] + "/qkv"
                if key not in self.wd:
                    self.wd[key] = torch.empty(cin, 3 * n, dtype=BF16, device=self.device)
                prep(self.wd[key], ld_dst=3 * n, col_offset={"to_q": 0, "to_k": n, "to_v": 2 * n}[leaf])
                continue
            taps = int(np.prod(shape[:-2])) if len(shape) == 4 else 1
            if base not in self.wd:
                self.wd[base] = torch.empty(cin, taps * n, dtype=BF16, device=self.device)
            if lora is not None:
                prep(self.wd[base])
            else:
                ops.prep_weight_dgrad(self.p(base + "/kernel"), self.wd[base], taps, cin, n)

    def g(self, name):
        off, shape = self.table[name]
        if self.lora_rank > 0:   # frozen: a scratch destination for the kernels that always write a parameter gradient
            return self._discard[int(name.endswith("/bias")), :int(np.prod(shape))].view(*shape)
        return self.grads[off:off + int(np.prod(shape))].view(*shape)

    # ----------------------------------------------------------------- context ----
    def prepare_context(self, ctx: torch.Tensor):
        """ctx fp32 [B, L, D]: computes every cross-attention K/V projection once.

        The bf16 context and the K/V buffers are allocated ONCE per context shape and reused: their addresses are baked
        into captured CUDA graphs (the sampler captures one denoising step and calls this method eagerly before every
        trajectory; the train steps capture this method itself), so a fresh allocation per call would leave a replayed
        graph reading the previous call's freed buffers."""
        b, l, d = ctx.shape
        cache = self._ctx_cache.get((b, l, d))
        if cache is None:
            cache = {"f32": torch.empty(b, l, d, dtype=F32, device=self.device),
                     "bf": torch.empty(b * l, d, dtype=BF16, device=self.device),
                     "kv": {key: torch.empty(b * l, w.shape[0], dtype=BF16, device=self.device)
                            for key, w in self.w.items() if key.endswith("attn2/kv")}}
            self._ctx_cache[(b, l, d)] = cache
        if ctx.data_ptr() != cache["f32"].data_ptr():
            cache["f32"].copy_(ctx)
        ctx_bf = cache["bf"]
        ops.cast_bf16(cache["f32"], ctx_bf)
        kv = cache["kv"]
        for key, out in kv.items():
            w = self.w[key]
            ops.igemm(a0=ctx_bf, wt=w, n=w.shape[0], c0=d, m=b * l, out_bf16=out)
        self.ctx_kv = kv
        self.ctx_batch = b
        self.ctx_len = l
        self._ctx_bf = ctx_bf
        return kv

    # ------------------------------------------------------------------ blocks ----
    def _resnet(self, name, x0, x1, c0, c1, cout, b, h, w, tape):
        A = self.arena
        hw, m, cin = h * w, b * h * w, c0 + c1
        has_sc = (name + "/conv_shortcut/kernel") in self.table
        assert has_sc or x1 is None
        gws = A.alloc((ops.groupnorm_workspace_floats(b, hw, cin),), F32)
        a = A.alloc((m, cin), BF16)
        raw = A.alloc((m, cin), BF16) if has_sc else None
        ops.groupnorm_fwd(x0, self.p(name + "/norm1/scale"), self.p(name + "/norm1/bias"), gws, b, hw, c0, x1=x1,
                          c1=c1, silu=True, y_bf16=a, raw_bf16=raw, stats0=_st(x0), stats1=_st(x1))
        tproj = self._tproj_views[name]          # computed by the grouped launch at the start of forward()
        hbuf = A.alloc_with_gn_stats((m, cout), hw)
        ops.igemm(a0=a, wt=self.w[name + "/conv1"], n=cout, c0=cin, conv=(b, h, w), taps=9,
                  bias=self.p(name + "/conv1/bias"), rowvec=tproj, rows_per_sample=hw, rowvec_ld=cout, out_f32=hbuf,
                  gn_stats=_st(hbuf))
        gws2 = A.alloc((ops.groupnorm_workspace_floats(b, hw, cout),), F32)
        a2 = A.alloc((m, cout), BF16)
        ops.groupnorm_fwd(hbuf, self.p(name + "/norm2/scale"), self.p(name + "/norm2/bias"), gws2, b, hw, cout,
                          silu=True, y_bf16=a2, stats0=_st(hbuf))
        if has_sc:
            sc = A.alloc((m, cout), F32)
            ops.igemm(a0=raw, wt=self.w[name + "/conv_shortcut"], n=cout, c0=cin, conv=(b, h, w), taps=1,
                      bias=self.p(name + "/conv_shortcut/bias"), out_f32=sc)
        else:
            sc = x0
        out = A.alloc_with_gn_stats((m, cout), hw)
        ops.igemm(a0=a2, wt=self.w[name + "/conv2"], n=cout, c0=cout, conv=(b, h, w), taps=9,
                  bias=self.p(name + "/conv2/bias"), residual=sc, out_f32=out, gn_stats=_st(out))
        if tape is None:
            for t in (gws, a, raw, tproj, hbuf, gws2, a2, sc if has_sc else None):
                A.release(t)
        else:
            tape.append(("resnet", dict(name=name, x0=x0, x1=x1, c0=c0, c1=c1, cout=cout, b=b, h=h, w=w, gws=gws,
                                        a=a, raw=raw, hbuf=hbuf, gws2=gws2, a2=a2, has_sc=has_sc, tproj=tproj,
                                        sc=sc if has_sc else None, out=out)))
        return out

    def _transformer(self, name, x, c, heads, b, h, w, tape):
        A = self.arena
        hw, m = h * w, b * h * w
        bl = name + "/transformer_blocks_0"
        L = self.ctx_len
        gws = A.alloc((ops.groupnorm_workspace_floats(b, hw, c),), F32)
        g = A.alloc((m, c), BF16)
        ops.groupnorm_fwd(x, self.p(name + "/norm/scale"), self.p(name + "/norm/bias"), gws, b, hw, c, silu=False,
                          y_bf16=g, stats0=_st(x))
        h0 = A.alloc((m, c), F32)
        ops.igemm(a0=g, wt=self.w[name + "/proj_in"], n=c, c0=c, m=m, bias=self.p(name + "/proj_in/bias"), out_f32=h0)
        # --- self attention
        ln1 = A.alloc((m, c), BF16)
        st1 = A.alloc((m, 2), F32)
        ops.layernorm_fwd(h0, self.p(bl + "/norm1/scale"), self.p(bl + "/norm1/bias"), ln1, m, c, stats=st1)
        qkv = A.alloc((m, 3 * c), BF16)
        ops.igemm(a0=ln1, wt=self.w[bl + "/attn1/qkv"], n=3 * c, c0=c, m=m, out_bf16=qkv)
        ao1 = A.alloc((m, c), BF16)
        lse1 = A.alloc((b, heads, hw), F32) if tape is not None else None
        ops.attention_fwd(qkv, qkv[:, c:], qkv[:, 2 * c:], ao1, b, heads, hw, hw, 3 * c, 3 * c, 3 * c, c, lse=lse1,
                          **_head_dim_kw(c, heads))
        h1 = A.alloc((m, c), F32)
        ops.igemm(a0=ao1, wt=self.w[bl + "/attn1/to_out_0"], n=c, c0=c, m=m, bias=self.p(bl + "/attn1/to_out_0/bias"),
                  residual=h0, out_f32=h1)
        # --- cross attention
        ln2 = A.alloc((m, c), BF16)
        st2 = A.alloc((m, 2), F32)
        ops.layernorm_fwd(h1, self.p(bl + "/norm2/scale"), self.p(bl + "/norm2/bias"), ln2, m, c, stats=st2)
        q2 = A.alloc((m, c), BF16)
        ops.igemm(a0=ln2, wt=self.w[bl + "/attn2/q"], n=c, c0=c, m=m, out_bf16=q2)
        kv = self.ctx_kv[bl + "/attn2/kv"]
        ao2 = A.alloc((m, c), BF16)
        lse2 = A.alloc((b, heads, hw), F32) if tape is not None else None
        ops.attention_fwd(q2, kv, kv[:, c:], ao2, b, heads, hw, L, c, 2 * c, 2 * c, c, lse=lse2,
                          **_head_dim_kw(c, heads))
        h2 = A.alloc((m, c), F32)
        ops.igemm(a0=ao2, wt=self.w[bl + "/attn2/to_out_0"], n=c, c0=c, m=m, bias=self.p(bl + "/attn2/to_out_0/bias"),
                  residual=h1, out_f32=h2)
        # --- GEGLU feed-forward
        ln3 = A.alloc((m, c), BF16)
        st3 = A.alloc((m, 2), F32)
        ops.layernorm_fwd(h2, self.p(bl + "/norm3/scale"), self.p(bl + "/norm3/bias"), ln3, m, c, stats=st3)
        ff = A.alloc((m, 4 * c), BF16)
        # training keeps the bf16 pre-activation (tile-interleaved [lin|gate]) for the GEGLU backward; the
        # activation itself always comes from the fp32 accumulators -> identical to the sampling forward
        ffpre = A.alloc((m, 8 * c), BF16) if tape is not None else None
        ops.igemm(a0=ln3, wt=self.w[bl + "/ff/net_0/proj"], n=8 * c, c0=c, m=m, bias=self.aux[bl + "/ff/net_0/proj"],
                  out_bf16=ff, geglu=True, bn=256, aux_bf16=ffpre)
        h3 = A.alloc((m, c), F32)
        h3b = A.alloc((m, c), BF16)
        ops.igemm(a0=ff, wt=self.w[bl + "/ff/net_2"], n=c, c0=4 * c, m=m, bias=self.p(bl + "/ff/net_2/bias"),
                  residual=h2, out_f32=h3, out_bf16=h3b)
        out = A.alloc_with_gn_stats((m, c), hw)
        ops.igemm(a0=h3b, wt=self.w[name + "/proj_out"], n=c, c0=c, m=m, bias=self.p(name + "/proj_out/bias"),
                  residual=x, out_f32=out, gn_stats=_st(out))
        if tape is None:
            for t in (gws, g, h0, ln1, st1, qkv, ao1, h1, ln2, st2, q2, ao2, h2, ln3, st3, ff, h3, h3b):
                A.release(t)
        else:
            tape.append(("transformer", dict(name=name, x=x, c=c, heads=heads, b=b, h=h, w=w, gws=gws, g=g, h0=h0,
                                             ln1=ln1, st1=st1, qkv=qkv, ao1=ao1, lse1=lse1, h1=h1, ln2=ln2, st2=st2,
                                             q2=q2, ao2=ao2, lse2=lse2, h2=h2, ln3=ln3, st3=st3, ffpre=ffpre, ff=ff,
                                             h3=h3, h3b=h3b, out=out)))
        return out

    # ----------------------------------------------------------------- forward ----
    def forward(self, latents: torch.Tensor, timesteps: torch.Tensor, out: Optional[torch.Tensor] = None,
                tape: Optional[list] = None, taps: Optional[dict] = None):
        """latents fp32 NCHW [B,4,H,W]; timesteps int32 [B] or [1]; returns eps fp32 NCHW [B,4,H,W].
        ``prepare_context`` must have been called with a context of the same batch size.
        ``tape``: list that receives what backward needs (training); ``taps``: debug dict name->tensor."""
        cfg, A = self.cfg, self.arena
        b, cin_lat, H, W = latents.shape
        assert self.ctx_kv is not None and self.ctx_batch == b, "prepare_context(ctx) with matching batch first"
        boc = cfg.block_out_channels
        te = cfg.time_embed_dim

        def tap(name, t, shape=None):
            if taps is not None:
                taps[name] = t.clone() if shape is None else t.view(*shape).clone()

        # time embedding: silu(temb) is what every consumer needs
        sincos = A.alloc((b, boc[0]), F32)
        ops.timestep_sincos(timesteps, sincos, b, boc[0])
        t1 = A.alloc((b, te), F32)
        ops.dense_small(sincos, self.p("time_embedding/linear_1/kernel"), self.p("time_embedding/linear_1/bias"), t1, b,
                        boc[0], te, silu_out=True)
        temb_act = A.alloc((b, te), F32)
        ops.dense_small(t1, self.p("time_embedding/linear_2/kernel"), self.p("time_embedding/linear_2/bias"), temb_act,
                        b, te, te, silu_out=True)
        tab = self._temb_tables.get(b)
        if tab is None:   # first (eager, pre-capture) pass at this batch size: offsets only, no addresses
            entries, views, y_off = [], [], 0
            for name in self._temb_names:
                w_off, wshape = self.table[name + "/time_emb_proj/kernel"]
                b_off, _ = self.table[name + "/time_emb_proj/bias"]
                n = int(wshape[1])
                entries.append((w_off, b_off, y_off, n))
                views.append((name, y_off, n))
                y_off += b * n
            dev_tab, ctas = ops.dense_small_group_table(entries, self.device)
            tab = self._temb_tables[b] = (dev_tab, ctas, views, y_off)
        dev_tab, ctas, views, total = tab
        tproj_all = A.alloc((total,), F32)
        ops.dense_small_grouped(temb_act, self.params, tproj_all, dev_tab, len(views), ctas, b, te)
        self._tproj_views = {name: tproj_all[o:o + b * n].view(b, n) for name, o, n in views}
        x = A.alloc_with_gn_stats((b * H * W, boc[0]), H * W)
        ops.conv_in(latents, self.p("conv_in/kernel"), self.p("conv_in/bias"), x, b, cin_lat, H, W, boc[0], gn_stats=_st(x))
        tap("conv_in", x, (b, H, W, boc[0]))
        if tape is not None:
            tape.append(("head", dict(latents=latents, sincos=sincos, t1=t1, temb_act=temb_act, b=b, H=H, W=W, x=x,
                                      tproj_all=tproj_all)))
            self._temb_act = temb_act
        skips = [(x, boc[0], H, W)]
        h, w, c_prev = H, W, boc[0]
        for i, c in enumerate(boc):
            for l in range(cfg.layers_per_block):
                name = f"down_blocks_{i}/resnets_{l}"
                y = self._resnet(name, x, None, c_prev, 0, c, b, h, w, tape)
                tap(name, y, (b, h, w, c))
                x, c_prev = y, c
                if cfg.down_has_attn[i]:
                    name = f"down_blocks_{i}/attentions_{l}"
                    y = self._transformer(name, x, c, cfg.attention_head_dim[i], b, h, w, tape)
                    tap(name, y, (b, h, w, c))
                    if tape is None:
                        A.release(x)  # resnet output is dead once the transformer consumed it (not a skip)
                    x = y
                skips.append((x, c, h, w))
            if i < len(boc) - 1:
                name = f"down_blocks_{i}/downsamplers_0"
                xb = A.alloc((b * h * w, c), BF16)
                ops.cast_bf16(x, xb)
                y = A.alloc_with_gn_stats((b * (h // 2) * (w // 2), c), (h // 2) * (w // 2))
                ops.igemm(a0=xb, wt=self.w[name + "/conv"], n=c, c0=c, conv=(b, h // 2, w // 2), taps=9, stride=2,
                          bias=self.p(name + "/conv/bias"), out_f32=y, gn_stats=_st(y))
                if tape is None:
                    A.release(xb)
                else:
                    tape.append(("down", dict(name=name, x=x, xb=xb, c=c, b=b, h=h, w=w, out=y)))
                h, w = h // 2, w // 2
                x = y
                tap(name, x, (b, h, w, c))
                skips.append((x, c, h, w))
        cm = boc[-1]
        y = self._resnet("mid_block/resnets_0", x, None, cm, 0, cm, b, h, w, tape)
        tap("mid_block/resnets_0", y, (b, h, w, cm))
        x = y
        y = self._transformer("mid_block/attentions_0", x, cm, cfg.attention_head_dim[-1], b, h, w, tape)
        tap("mid_block/attentions_0", y, (b, h, w, cm))
        if tape is None:
            A.release(x)
        x = y
        y = self._resnet("mid_block/resnets_1", x, None, cm, 0, cm, b, h, w, tape)
        tap("mid_block/resnets_1", y, (b, h, w, cm))
        if tape is None:
            A.release(x)
        x = y
        rev = tuple(reversed(boc))
        rev_heads = tuple(reversed(cfg.attention_head_dim))
        has_attn = tuple(reversed(cfg.down_has_attn))
        c_prev = rev[0]
        for i, c in enumerate(rev):
            for l in range(cfg.layers_per_block + 1):
                sk, sc_, sh, sw = skips.pop()
                assert (sh, sw) == (h, w)
                name = f"up_blocks_{i}/resnets_{l}"
                y = self._resnet(name, x, sk, c_prev, sc_, c, b, h, w, tape)
                tap(name, y, (b, h, w, c))
                if tape is None:
                    A.release(x)
                    A.release(sk)
                x, c_prev = y, c
                if has_attn[i]:
                    name = f"up_blocks_{i}/attentions_{l}"
                    y = self._transformer(name, x, c, rev_heads[i], b, h, w, tape)
                    tap(name, y, (b, h, w, c))
                    if tape is None:
                        A.release(x)
                    x = y
            if i < len(rev) - 1:
                name = f"up_blocks_{i}/upsamplers_0"
                up = A.alloc((b * 4 * h * w, c), BF16)
                ops.upsample2x_bf16(x, up, b, h, w, c)
                y = A.alloc_with_gn_stats((b * 4 * h * w, c), 4 * h * w)
                ops.igemm(a0=up, wt=self.w[name + "/conv"], n=c, c0=c, conv=(b, 2 * h, 2 * w), taps=9,
                          bias=self.p(name + "/conv/bias"), out_f32=y, gn_stats=_st(y))
                if tape is None:
                    A.release(up)
                    A.release(x)
                else:
                    tape.append(("up", dict(name=name, x=x, up=up, c=c, b=b, h=h, w=w, out=y)))
                h, w = 2 * h, 2 * w
                x = y
                tap(name, x, (b, h, w, c))
        c0 = boc[0]
        gws = A.alloc((ops.groupnorm_workspace_floats(b, h * w, c0),), F32)
        yf = A.alloc((b * h * w, c0), F32)
        ops.groupnorm_fwd(x, self.p("conv_norm_out/scale"), self.p("conv_norm_out/bias"), gws, b, h * w, c0, silu=True,
                          y_f32=yf, stats0=_st(x))
        if out is None:
            out = torch.empty(b, cfg.out_channels, h, w, dtype=F32, device=self.device)
        ops.conv_out(yf, self.p("conv_out/kernel"), self.p("conv_out/bias"), out, b, h, w, c0, cfg.out_channels)
        if tape is None:
            for t in (gws, yf, x, sincos, t1, temb_act, tproj_all):
                A.release(t)
        else:
            tape.append(("tail", dict(x=x, gws=gws, yf=yf, b=b, h=h, w=w, c=c0)))
        return out

    # ---------------------------------------------------------------- backward ----
    def backward(self, tape: list, d_eps: torch.Tensor):
        """Back-propagates d(loss)/d(eps) [B,4,H,W] through the taped forward; parameter gradients are
        ACCUMULATED into ``self.grads`` (AccumulatingTrainState semantics).  Releases the tape's buffers.
        In LoRA mode every data gradient is computed exactly as in full fine-tuning, no base-parameter gradient is
        formed (no weight-gradient GEMMs, bias sums or time-embedding chain), and the adapter gradients are
        accumulated into ``self.lora_grads`` (ops.lora_grad)."""
        assert self.train_mode and (self.grads is not None or self.lora_rank > 0)
        full = self.lora_rank == 0
        A = self.arena
        grads: Dict[int, torch.Tensor] = {}

        def put(x, d, m, c, lds=None):
            """register contribution d [m, c] (row pitch lds) to the gradient of stream tensor x"""
            if id(x) in grads:
                ops.copy2d(d, lds or c, grads[id(x)], c, m, c, accumulate=True)
                return False  # caller still owns d
            if lds is None or lds == c:
                grads[id(x)] = d
                return True   # ownership moved
            t = A.alloc((m, c), F32)
            ops.copy2d(d, lds, t, c, m, c, accumulate=False)
            grads[id(x)] = t
            return False

        temb_state = {"d": None}

        def bias_grad_and_cast(dy, m, n, bias_names):
            dyb = A.alloc((m, n), BF16)
            if not full:                       # frozen biases: the bf16 copy only
                ops.cast_bf16(dy, dyb)
            elif len(bias_names) == 1:
                ops.colsum_cast(dy, m, n, y_bf16=dyb, out=self.g(bias_names[0]).view(1, n), accumulate=True)
            else:
                tmp = A.alloc((1, n), F32)
                ops.colsum_cast(dy, m, n, y_bf16=dyb, out=tmp, accumulate=False)
                for nm in bias_names:
                    ops.copy2d(tmp, n, self.g(nm).view(1, n), n, 1, n, accumulate=True)
                A.release(tmp)
            return dyb

        for kind, r in reversed(tape):
            if kind == "tail":
                b, h, w, c = r["b"], r["h"], r["w"], r["c"]
                m = b * h * w
                d_yf = A.alloc((m, c), F32)
                ops.conv_out_bwd(r["yf"], self.p("conv_out/kernel"), d_eps, d_yf, self.g("conv_out/kernel"),
                                 self.g("conv_out/bias"), b, h, w, c)
                dx = A.alloc((m, c), F32)
                ops.groupnorm_bwd(r["x"], self.p("conv_norm_out/scale"), self.p("conv_norm_out/bias"), r["gws"], b, h * w,
                                  c, d_yf, dx, self.g("conv_norm_out/scale"), self.g("conv_norm_out/bias"), silu=True)
                grads[id(r["x"])] = dx
                for t in (d_yf, r["yf"], r["gws"]):
                    A.release(t)
            elif kind == "up":
                name, b, h, w, c = r["name"], r["b"], r["h"], r["w"], r["c"]
                m2 = b * 4 * h * w
                dy = grads.pop(id(r["out"]))
                dyb = bias_grad_and_cast(dy, m2, c, [name + "/conv/bias"])
                if full:
                    ops.wgrad(dy=dyb, n=c, x0=r["up"], c0=c, conv=(b, 2 * h, 2 * w), taps=9,
                              dw=self.g(name + "/conv/kernel"))
                d_up = A.alloc((m2, c), F32)
                ops.igemm(a0=dyb, wt=self.wd[name + "/conv"], n=c, c0=c, conv=(b, 2 * h, 2 * w), taps=9, out_f32=d_up)
                if id(r["x"]) in grads:
                    ops.upsample2x_bwd(d_up, grads[id(r["x"])], b, h, w, c, accumulate=True)
                else:
                    dx = A.alloc((b * h * w, c), F32)
                    ops.upsample2x_bwd(d_up, dx, b, h, w, c, accumulate=False)
                    grads[id(r["x"])] = dx
                for t in (dy, dyb, d_up, r["up"], r["out"]):
                    A.release(t)
            elif kind == "down":
                name, b, h, w, c = r["name"], r["b"], r["h"], r["w"], r["c"]
                mo = b * (h // 2) * (w // 2)
                dy = grads.pop(id(r["out"]))
                dyb = bias_grad_and_cast(dy, mo, c, [name + "/conv/bias"])
                if full:
                    ops.wgrad(dy=dyb, n=c, x0=r["xb"], c0=c, conv=(b, h // 2, w // 2), taps=9, stride=2,
                              dw=self.g(name + "/conv/kernel"))
                dil = A.alloc((b * h * w, c), BF16)
                ops.dilate2x_bf16(dy, dil, b, h // 2, w // 2, c)
                if id(r["x"]) in grads:
                    ops.igemm(a0=dil, wt=self.wd[name + "/conv"], n=c, c0=c, conv=(b, h, w), taps=9,
                              out_f32=grads[id(r["x"])], accumulate=True)
                else:
                    dx = A.alloc((b * h * w, c), F32)
                    ops.igemm(a0=dil, wt=self.wd[name + "/conv"], n=c, c0=c, conv=(b, h, w), taps=9, out_f32=dx)
                    grads[id(r["x"])] = dx
                for t in (dy, dyb, dil, r["xb"], r["out"]):
                    A.release(t)
            elif kind == "resnet":
                self._resnet_bwd(r, grads, put, bias_grad_and_cast, temb_state)
            elif kind == "transformer":
                self._transformer_bwd(r, grads, put, bias_grad_and_cast)
            elif kind == "head":
                b, H, W = r["b"], r["H"], r["W"]
                c0 = self.cfg.block_out_channels[0]
                te = self.cfg.time_embed_dim
                x = r.get("x")
                dx = grads.pop(id(x))
                if full:
                    ops.colsum_cast(dx, b * H * W, c0, out=self.g("conv_in/bias").view(1, c0), accumulate=True)
                    ops.conv_in_wgrad(r["latents"], dx, self.g("conv_in/kernel"), b, self.cfg.in_channels, H, W, c0)
                A.release(dx)
                A.release(x)
                d_temb = temb_state["d"]
                if d_temb is not None:
                    dpre = A.alloc((b, te), F32)
                    d_t1 = A.alloc((b, te), F32)
                    ops.dense_small_bwd(r["t1"], self.p("time_embedding/linear_2/kernel"),
                                        self.p("time_embedding/linear_2/bias"), d_temb, dpre,
                                        self.g("time_embedding/linear_2/kernel"), self.g("time_embedding/linear_2/bias"),
                                        d_t1, b, te, te, silu_out=True)
                    ops.dense_small_bwd(r["sincos"], self.p("time_embedding/linear_1/kernel"),
                                        self.p("time_embedding/linear_1/bias"), d_t1, dpre,
                                        self.g("time_embedding/linear_1/kernel"), self.g("time_embedding/linear_1/bias"),
                                        None, b, c0, te, silu_out=True)
                    for t in (dpre, d_t1, d_temb):
                        A.release(t)
                for t in (r["sincos"], r["t1"], r["temb_act"], r["tproj_all"]):
                    A.release(t)
        assert not grads, f"{len(grads)} stream gradients were never consumed"

    def _resnet_bwd(self, r, grads, put, bias_grad_and_cast, temb_state):
        A = self.arena
        name, b, h, w = r["name"], r["b"], r["h"], r["w"]
        c0, c1, cout = r["c0"], r["c1"], r["cout"]
        cin, hw, m = c0 + c1, h * w, b * h * w
        te = self.cfg.time_embed_dim
        dy = grads.pop(id(r["out"]))
        if getattr(self, "_dbg", None) is not None:
            self._dbg[name] = dy.clone()
        full = self.lora_rank == 0
        names = [name + "/conv2/bias"] + ([name + "/conv_shortcut/bias"] if r["has_sc"] else [])
        dyb = bias_grad_and_cast(dy, m, cout, names)
        if full:
            ops.wgrad(dy=dyb, n=cout, x0=r["a2"], c0=cout, conv=(b, h, w), taps=9, dw=self.g(name + "/conv2/kernel"))
        # gradients that go straight from a dgrad GEMM into a norm's backward travel as bf16 (half the bytes on both sides;
        # the forward value they belong to was itself a bf16 GEMM operand)
        d_a2 = A.alloc((m, cout), BF16)
        ops.igemm(a0=dyb, wt=self.wd[name + "/conv2"], n=cout, c0=cout, conv=(b, h, w), taps=9, out_bf16=d_a2)
        d_h = A.alloc((m, cout), F32)
        ops.groupnorm_bwd(r["hbuf"], self.p(name + "/norm2/scale"), self.p(name + "/norm2/bias"), r["gws2"], b, hw, cout,
                          d_a2, d_h, self.g(name + "/norm2/scale"), self.g(name + "/norm2/bias"), silu=True)
        A.release(d_a2)
        # h = conv1(a) + bias1 + time_emb_proj(silu(temb))[b]
        d_hb = A.alloc((m, cout), BF16)
        if full:
            d_tproj = A.alloc((b, cout), F32)
            ops.colsum_cast(d_h, m, cout, y_bf16=d_hb, out=d_tproj, rows_per_group=hw, accumulate=False)
            A.release(d_h)
            ops.colsum_cast(d_tproj, b, cout, out=self.g(name + "/conv1/bias").view(1, cout), accumulate=True)
            first = temb_state["d"] is None
            if first:
                temb_state["d"] = A.alloc((b, te), F32)
            dpre = A.alloc((b, cout), F32)
            ops.dense_small_bwd(self._temb_act, self.p(name + "/time_emb_proj/kernel"), None, d_tproj, dpre,
                                self.g(name + "/time_emb_proj/kernel"), self.g(name + "/time_emb_proj/bias"),
                                temb_state["d"], b, te, cout, dx_accumulate=not first)
            A.release(dpre)
            A.release(d_tproj)
            ops.wgrad(dy=d_hb, n=cout, x0=r["a"], c0=cin, conv=(b, h, w), taps=9, dw=self.g(name + "/conv1/kernel"))
        else:                                  # frozen time embedding: no d_tproj, no chain into temb
            ops.cast_bf16(d_h, d_hb)
            A.release(d_h)
        d_a = A.alloc((m, cin), BF16)
        ops.igemm(a0=d_hb, wt=self.wd[name + "/conv1"], n=cin, c0=cout, conv=(b, h, w), taps=9, out_bf16=d_a)
        A.release(d_hb)
        if r["has_sc"]:
            if full:
                ops.wgrad(dy=dyb, n=cout, x0=r["raw"], c0=cin, conv=(b, h, w), taps=1,
                          dw=self.g(name + "/conv_shortcut/kernel"))
            dcat = A.alloc((m, cin), F32)
            ops.igemm(a0=dyb, wt=self.wd[name + "/conv_shortcut"], n=cin, c0=cout, conv=(b, h, w), taps=1, out_f32=dcat)
            ops.groupnorm_bwd(r["x0"], self.p(name + "/norm1/scale"), self.p(name + "/norm1/bias"), r["gws"], b, hw, c0,
                              d_a, dcat, self.g(name + "/norm1/scale"), self.g(name + "/norm1/bias"), x1=r["x1"], c1=c1,
                              dx1=dcat[:, c0:] if c1 else None, silu=True, accumulate=True, ldd0=cin, ldd1=cin)
            if c1 == 0:
                if not put(r["x0"], dcat, m, cin):
                    A.release(dcat)
            else:
                put(r["x0"], dcat, m, c0, lds=cin)
                put(r["x1"], dcat[:, c0:], m, c1, lds=cin)
                A.release(dcat)
            A.release(dy)
        else:
            if id(r["x0"]) in grads:
                tgt = grads[id(r["x0"])]
                ops.copy2d(dy, cout, tgt, cout, m, cout, accumulate=True)
                A.release(dy)
            else:
                tgt = dy
                grads[id(r["x0"])] = dy
            ops.groupnorm_bwd(r["x0"], self.p(name + "/norm1/scale"), self.p(name + "/norm1/bias"), r["gws"], b, hw, c0,
                              d_a, tgt, self.g(name + "/norm1/scale"), self.g(name + "/norm1/bias"), silu=True,
                              accumulate=True)
        A.release(d_a)
        A.release(dyb)
        for t in (r["gws"], r["a"], r["raw"], r["hbuf"], r["gws2"], r["a2"], r["tproj"], r["sc"], r["out"]):
            A.release(t)

    def _transformer_bwd(self, t, grads, put, bias_grad_and_cast):
        A = self.arena
        name, b, h, w, c, heads = t["name"], t["b"], t["h"], t["w"], t["c"], t["heads"]
        hw, m = h * w, b * h * w
        bl = name + "/transformer_blocks_0"
        L = self.ctx_len
        dctx = self.cfg.cross_attention_dim
        full = self.lora_rank == 0

        def lora_grad(x, dys, ld, projs, attn, mm, k):
            """adapter gradients of the projections ``projs`` of ``attn``, which share the input x [mm, k]"""
            bases = [f"{bl}/{attn}/{p}" for p in projs]
            ops.lora_grad(x, dys, [self.lp(b_ + "/lora_down") for b_ in bases], [self.lp(b_ + "/lora_up") for b_ in bases],
                          [self.lg(b_ + "/lora_down") for b_ in bases], [self.lg(b_ + "/lora_up") for b_ in bases],
                          mm, k, c, self.lora_rank, lddy=ld)
        dy = grads.pop(id(t["out"]))
        if getattr(self, "_dbg", None) is not None:
            self._dbg[name] = dy.clone()
        # out = proj_out(h3b) + x
        dyb = bias_grad_and_cast(dy, m, c, [name + "/proj_out/bias"])
        if full:
            ops.wgrad(dy=dyb, n=c, x0=t["h3b"], c0=c, m=m, dw=self.g(name + "/proj_out/kernel").view(c, c))
        d_h = A.alloc((m, c), F32)   # running gradient of the transformer-internal residual stream
        ops.igemm(a0=dyb, wt=self.wd[name + "/proj_out"], n=c, c0=c, m=m, out_f32=d_h)
        A.release(dyb)
        x_owned = put(t["x"], dy, m, c)
        if not x_owned:
            A.release(dy)
        # h3 = ff2(ff) + h2
        d3b = bias_grad_and_cast(d_h, m, c, [bl + "/ff/net_2/bias"])
        if full:
            ops.wgrad(dy=d3b, n=c, x0=t["ff"], c0=4 * c, m=m, dw=self.g(bl + "/ff/net_2/kernel"))
        d_ff = A.alloc((m, 4 * c), BF16)
        ops.igemm(a0=d3b, wt=self.wd[bl + "/ff/net_2"], n=4 * c, c0=c, m=m, out_bf16=d_ff)
        A.release(d3b)
        d_pre = A.alloc((m, 8 * c), BF16)
        ops.geglu_bwd(t["ffpre"], d_ff, d_pre, m, 8 * c, 256)
        A.release(d_ff)
        if full:
            ops.colsum_bf16(d_pre, m, 8 * c, self.g(bl + "/ff/net_0/proj/bias").view(1, 8 * c), accumulate=True)
            ops.wgrad(dy=d_pre, n=8 * c, x0=t["ln3"], c0=c, m=m, dw=self.g(bl + "/ff/net_0/proj/kernel"))
        d_ln = A.alloc((m, c), BF16)   # dgrad GEMM -> norm backward: bf16 (see _resnet_bwd)
        ops.igemm(a0=d_pre, wt=self.wd[bl + "/ff/net_0/proj"], n=c, c0=8 * c, m=m, out_bf16=d_ln)
        A.release(d_pre)
        lws = A.alloc((ops.layernorm_bwd_workspace_floats(m, c),), F32)
        ops.layernorm_bwd(t["h2"], self.p(bl + "/norm3/scale"), t["st3"], d_ln, d_h, self.g(bl + "/norm3/scale"),
                          self.g(bl + "/norm3/bias"), lws, m, c, accumulate=True)
        # h2 = out2(ao2) + h1   (cross attention)
        d2b = bias_grad_and_cast(d_h, m, c, [bl + "/attn2/to_out_0/bias"])
        if full:
            ops.wgrad(dy=d2b, n=c, x0=t["ao2"], c0=c, m=m, dw=self.g(bl + "/attn2/to_out_0/kernel"))
        else:
            lora_grad(t["ao2"], [d2b], c, ["to_out_0"], "attn2", m, c)
        d_ao = A.alloc((m, c), BF16)
        ops.igemm(a0=d2b, wt=self.wd[bl + "/attn2/to_out_0"], n=c, c0=c, m=m, out_bf16=d_ao)
        A.release(d2b)
        kv = self.ctx_kv[bl + "/attn2/kv"]
        dq2 = A.alloc((m, c), BF16)
        dkv = A.alloc((b * L, 2 * c), BF16)
        delta = A.alloc((b, heads, hw), F32)
        ops.attention_bwd(t["q2"], kv, kv[:, c:], t["ao2"], d_ao, t["lse2"], delta, dq2, dkv, dkv[:, c:], b, heads, hw, L,
                          c, 2 * c, 2 * c, c, c, c, 2 * c, 2 * c, **_head_dim_kw(c, heads))
        if full:
            ops.wgrad(dy=dq2, n=c, x0=t["ln2"], c0=c, m=m, dw=self.g(bl + "/attn2/to_q/kernel"))
            ops.wgrad(dy=dkv, ldy=2 * c, n=c, x0=self._ctx_bf, c0=dctx, m=b * L, dw=self.g(bl + "/attn2/to_k/kernel"))
            ops.wgrad(dy=dkv[:, c:], ldy=2 * c, n=c, x0=self._ctx_bf, c0=dctx, m=b * L,
                      dw=self.g(bl + "/attn2/to_v/kernel"))
        else:
            lora_grad(t["ln2"], [dq2], c, ["to_q"], "attn2", m, c)
            lora_grad(self._ctx_bf, [dkv, dkv[:, c:]], 2 * c, ["to_k", "to_v"], "attn2", b * L, dctx)
        ops.igemm(a0=dq2, wt=self.wd[bl + "/attn2/to_q"], n=c, c0=c, m=m, out_bf16=d_ln)
        ops.layernorm_bwd(t["h1"], self.p(bl + "/norm2/scale"), t["st2"], d_ln, d_h, self.g(bl + "/norm2/scale"),
                          self.g(bl + "/norm2/bias"), lws, m, c, accumulate=True)
        A.release(dq2)
        A.release(dkv)
        # h1 = out1(ao1) + h0   (self attention)
        d1b = bias_grad_and_cast(d_h, m, c, [bl + "/attn1/to_out_0/bias"])
        if full:
            ops.wgrad(dy=d1b, n=c, x0=t["ao1"], c0=c, m=m, dw=self.g(bl + "/attn1/to_out_0/kernel"))
        else:
            lora_grad(t["ao1"], [d1b], c, ["to_out_0"], "attn1", m, c)
        ops.igemm(a0=d1b, wt=self.wd[bl + "/attn1/to_out_0"], n=c, c0=c, m=m, out_bf16=d_ao)
        A.release(d1b)
        qkv = t["qkv"]
        dqkv = A.alloc((m, 3 * c), BF16)
        ops.attention_bwd(qkv, qkv[:, c:], qkv[:, 2 * c:], t["ao1"], d_ao, t["lse1"], delta, dqkv, dqkv[:, c:],
                          dqkv[:, 2 * c:], b, heads, hw, hw, 3 * c, 3 * c, 3 * c, c, c, 3 * c, 3 * c, 3 * c,
                          **_head_dim_kw(c, heads))
        if full:
            for i, nm in enumerate(("to_q", "to_k", "to_v")):
                ops.wgrad(dy=dqkv[:, i * c:], ldy=3 * c, n=c, x0=t["ln1"], c0=c, m=m,
                          dw=self.g(f"{bl}/attn1/{nm}/kernel"))
        else:
            lora_grad(t["ln1"], [dqkv, dqkv[:, c:], dqkv[:, 2 * c:]], 3 * c, ["to_q", "to_k", "to_v"], "attn1", m, c)
        ops.igemm(a0=dqkv, c0=3 * c, wt=self.wd[bl + "/attn1/qkv"], n=c, m=m, out_bf16=d_ln)   # one GEMM over K = 3C
        ops.layernorm_bwd(t["h0"], self.p(bl + "/norm1/scale"), t["st1"], d_ln, d_h, self.g(bl + "/norm1/scale"),
                          self.g(bl + "/norm1/bias"), lws, m, c, accumulate=True)
        for z in (dqkv, d_ao, delta, lws):
            A.release(z)
        # h0 = proj_in(g)
        d0b = bias_grad_and_cast(d_h, m, c, [name + "/proj_in/bias"])
        if full:
            ops.wgrad(dy=d0b, n=c, x0=t["g"], c0=c, m=m, dw=self.g(name + "/proj_in/kernel").view(c, c))
        ops.igemm(a0=d0b, wt=self.wd[name + "/proj_in"], n=c, c0=c, m=m, out_bf16=d_ln)
        A.release(d0b)
        A.release(d_h)
        ops.groupnorm_bwd(t["x"], self.p(name + "/norm/scale"), self.p(name + "/norm/bias"), t["gws"], b, hw, c, d_ln,
                          grads[id(t["x"])], self.g(name + "/norm/scale"), self.g(name + "/norm/bias"), silu=False,
                          accumulate=True)
        A.release(d_ln)
        for key in ("gws", "g", "h0", "ln1", "st1", "qkv", "ao1", "lse1", "h1", "ln2", "st2", "q2", "ao2", "lse2", "h2",
                    "ln3", "st3", "ffpre", "ff", "h3", "h3b", "out"):
            A.release(t[key])
