"""SD1.x support without a GPU: the U-Net host assembly at head dims 40, 80 and 160 with 1x1-conv projections, run on
the torch-CPU emulation of the ops (tests/_cpu_ops_emulator.py, with attention at any head dim) against the oracle; the
model registry for the SD1 ids and their text tower; and an SD1-layout diffusers checkpoint directory through
utils/pretrained.py."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ddpo_b200 import unet_spec  # noqa: E402
from ddpo_b200.unet_spec import UNetConfig  # noqa: E402

SD1_IDS = ["duongna/stable-diffusion-v1-4-flax", "CompVis/stable-diffusion-v1-4", "runwayml/stable-diffusion-v1-5"]

# SD1 topology at one width: 320 channels over (8, 4, 2, 2) heads reaches head dims 40, 80 and 160 (160 also in the
# mid block), with SD1's 768-wide context and 1x1-conv proj_in / proj_out
SD1_SMALL = UNetConfig(block_out_channels=(320, 320, 320, 320), attention_head_dim=(8, 4, 2, 2), cross_attention_dim=768,
                       use_linear_projection=False, sample_size=16)


class _EmulatedOps:
    """the torch-CPU emulation of the ops (tests/_cpu_ops_emulator.py) with attention at any head dim: head h of
    q/k/v/out at columns [h*d, h*d + d), scale d^-0.5, P rounded to bf16 before P V as the kernel does"""

    def __init__(self):
        import _cpu_ops_emulator as E
        self._e = E

    def __getattr__(self, name):
        return getattr(self._e, name)

    @staticmethod
    def _heads(t, n, batch, heads, d):
        return t[:, :heads * d].reshape(batch, n, heads, d).permute(0, 2, 1, 3).float()

    def attention_fwd(self, q, k, v, out, batch, heads, nq, nk, ldq, ldk, ldv, ldo, lse=None, causal=False, head_dim=64):
        d = head_dim
        qq, kk, vv = self._heads(q, nq, batch, heads, d), self._heads(k, nk, batch, heads, d), self._heads(v, nk, batch, heads, d)
        s = qq @ kk.transpose(-1, -2) * d ** -0.5
        if causal:
            s = s + torch.full((nq, nk), float("-inf")).triu(1)
        p = torch.softmax(s, -1).to(torch.bfloat16).float()
        out[:, :heads * d].copy_((p @ vv).permute(0, 2, 1, 3).reshape(batch * nq, heads * d).to(torch.bfloat16))

    def attention_bwd(self, q, k, v, out, dout, lse, delta, dq, dk, dv, batch, heads, nq, nk, ldq, ldk, ldv, ldo, lddo, lddq,
                      lddk, lddv, head_dim=64):
        d = head_dim
        qq, kk, vv = (self._heads(t, n, batch, heads, d).requires_grad_(True) for t, n in ((q, nq), (k, nk), (v, nk)))
        o = torch.softmax(qq @ kk.transpose(-1, -2) * d ** -0.5, -1) @ vv
        o.backward(self._heads(dout, nq, batch, heads, d))
        back = lambda t, n: t.permute(0, 2, 1, 3).reshape(batch * n, heads * d).to(torch.bfloat16)
        dq[:, :heads * d] = back(qq.grad, nq)
        dk[:, :heads * d] = back(kk.grad, nk)
        dv[:, :heads * d] = back(vv.grad, nk)


def _net(monkeypatch, cfg, flat):
    import _cpu_ops_emulator as E
    from ddpo_b200 import unet as U
    monkeypatch.setattr(U, "ops", _EmulatedOps())
    monkeypatch.setattr(U, "Arena", E.CpuArena)
    return U.UNet(cfg, flat, device="cpu")


def test_emulated_attention_at_64_is_the_emulator():
    """the wrapper's attention at d = 64 gives the emulator's bits, so the SD1 dry runs use the SD2 dry runs' reference"""
    import _cpu_ops_emulator as E
    g = torch.Generator().manual_seed(3)
    b, n, heads, c = 2, 16, 2, 128
    qkv = torch.randn(b * n, 3 * c, generator=g).to(torch.bfloat16)
    do = torch.randn(b * n, c, generator=g).to(torch.bfloat16)
    outs = []
    for ops in (E, _EmulatedOps()):
        out = torch.zeros(b * n, c, dtype=torch.bfloat16)
        ops.attention_fwd(qkv, qkv[:, c:], qkv[:, 2 * c:], out, b, heads, n, n, 3 * c, 3 * c, 3 * c, c)
        dqkv = torch.zeros(b * n, 3 * c, dtype=torch.bfloat16)
        ops.attention_bwd(qkv, qkv[:, c:], qkv[:, 2 * c:], out, do, None, None, dqkv, dqkv[:, c:], dqkv[:, 2 * c:], b, heads,
                          n, n, 3 * c, 3 * c, 3 * c, c, c, 3 * c, 3 * c, 3 * c)
        outs.append((out, dqkv))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_sd1_small_reaches_every_sd1_head_dim():
    dims = {c // h for c, h in zip(SD1_SMALL.block_out_channels, SD1_SMALL.attention_head_dim)}
    assert dims == {40, 80, 160}
    assert {c // 8 for c in unet_spec.SD1.block_out_channels} == {40, 80, 160}
    table, _ = unet_spec.param_offsets(SD1_SMALL)
    assert table["down_blocks_0/attentions_0/proj_in/kernel"][1] == (1, 1, 320, 320)


def test_unsupported_head_dim_is_refused_with_a_message():
    from ddpo_b200 import unet as U
    cfg = UNetConfig(block_out_channels=(384, 384, 384, 384), attention_head_dim=(8, 8, 8, 8), cross_attention_dim=768,
                     use_linear_projection=False, sample_size=16)       # head dim 48
    with pytest.raises(AssertionError, match="head dims"):
        U.UNet(cfg, torch.zeros(unet_spec.param_offsets(cfg)[1]), device="cpu")


def test_sd1_forward_host_assembly_matches_oracle(monkeypatch):
    from oracle.unet import UNetOracle
    cfg, batch = SD1_SMALL, 2
    flat = unet_spec.init_flat_params(cfg, 0)
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(batch, 4, cfg.sample_size, cfg.sample_size, generator=g)
    ctx = torch.randn(batch, cfg.ctx_len, cfg.cross_attention_dim, generator=g)
    ts = torch.tensor([981, 21], dtype=torch.int32)
    net = _net(monkeypatch, cfg, flat)
    net.prepare_context(ctx)
    eps = net.forward(lat, ts)
    with torch.no_grad():
        ref = UNetOracle(cfg, unet_spec.views(flat, cfg))(lat, ts.long(), ctx)
    rel = ((eps - ref).norm() / ref.norm()).item()
    assert eps.shape == ref.shape and rel < 2e-2, rel


def test_sd1_backward_host_assembly_matches_oracle_autograd(monkeypatch):
    from oracle.unet import UNetOracle
    cfg, batch = SD1_SMALL, 2
    flat = unet_spec.init_flat_params(cfg, 0)
    g = torch.Generator().manual_seed(11)
    s = cfg.sample_size
    lat = torch.randn(batch, 4, s, s, generator=g)
    ctx = torch.randn(batch, cfg.ctx_len, cfg.cross_attention_dim, generator=g)
    ts = torch.tensor([981, 21], dtype=torch.int32)
    d_eps = torch.randn(batch, 4, s, s, generator=g) / (4 * s * s)
    net = _net(monkeypatch, cfg, flat)
    net.enable_training()
    net.prepare_context(ctx)
    tape = []
    net.forward(lat, ts, tape=tape)
    net.backward(tape, d_eps)
    params = {k: v.clone().requires_grad_(True) for k, v in unet_spec.views(flat, cfg).items()}
    UNetOracle(cfg, params)(lat, ts.long(), ctx).backward(d_eps)
    table, _ = unet_spec.param_offsets(cfg)
    ref = torch.zeros_like(flat)
    for name, (off, shape) in table.items():
        if params[name].grad is not None:
            ref[off:off + params[name].numel()] = params[name].grad.reshape(-1)
    tot = ((net.grads - ref).norm() / ref.norm()).item()
    assert tot < 4e-2, tot
    worst = 0.0
    for name, (off, shape) in table.items():
        n = int(np.prod(shape))
        a, r = net.grads[off:off + n], ref[off:off + n]
        if r.norm() > 1e-3 * ref.norm() / np.sqrt(len(table)):
            worst = max(worst, ((a - r).norm() / r.norm()).item())
    assert worst < 0.2, worst
    for blk in ("down_blocks_1/attentions_0", "mid_block/attentions_0"):       # the 1x1-conv projections get gradients
        for proj in ("proj_in", "proj_out"):
            off, shape = table[f"{blk}/{proj}/kernel"]
            n = int(np.prod(shape))
            a, r = net.grads[off:off + n], ref[off:off + n]
            assert r.norm() > 0 and ((a - r).norm() / r.norm()).item() < 0.2, (blk, proj)


@pytest.mark.parametrize("model_id", SD1_IDS)
def test_sd1_ids_resolve_to_sd1_with_the_clip_l_text_tower(model_id):
    from ddpo_b200.text_encoder import text_config_for
    from ddpo_b200.utils.serialization import unet_config_for
    assert unet_config_for(model_id) is unet_spec.SD1
    assert text_config_for(model_id).hidden_size == unet_spec.SD1.cross_attention_dim == 768
    assert text_config_for(model_id).hidden_act == "quick_gelu"


def test_sd2_ids_keep_their_text_tower():
    from ddpo_b200.text_encoder import SD2_TEXT, text_config_for
    from ddpo_b200.utils.serialization import unet_config_for
    assert unet_config_for("stabilityai/stable-diffusion-2-base") is unet_spec.SD2_BASE
    assert text_config_for("stabilityai/stable-diffusion-2-base") is SD2_TEXT


def test_sd1_layout_diffusers_directory_loads(tmp_path):
    """diffusers' SD1 unet/config.json has a scalar attention_head_dim and no use_linear_projection key; its PyTorch
    weights hold proj_in / proj_out as OIHW [C, C, 1, 1] convolutions"""
    from safetensors.torch import save_file
    from _torch_twin import UNet2DConditionTwin, load_flax_params
    from ddpo_b200.utils import pretrained as P
    cfg = UNetConfig(block_out_channels=(320, 320, 320, 320), attention_head_dim=(8, 8, 8, 8), cross_attention_dim=768,
                     use_linear_projection=False, sample_size=16)
    flat = unet_spec.init_flat_params(cfg, 7)
    views = unet_spec.views(flat, cfg)
    d = tmp_path / "ckpt"
    os.makedirs(d / "unet")
    with open(d / "unet" / "config.json", "w") as f:
        json.dump({"block_out_channels": list(cfg.block_out_channels), "attention_head_dim": 8,
                   "cross_attention_dim": 768, "sample_size": cfg.sample_size, "layers_per_block": cfg.layers_per_block,
                   "in_channels": 4, "out_channels": 4,
                   "down_block_types": ["CrossAttnDownBlock2D"] * 3 + ["DownBlock2D"]}, f)
    twin = load_flax_params(UNet2DConditionTwin(cfg), views)
    sd = {k: v.contiguous() for k, v in twin.state_dict().items()}
    assert tuple(sd["down_blocks.0.attentions.0.proj_in.weight"].shape) == (320, 320, 1, 1)
    save_file(sd, str(d / "unet" / "diffusion_pytorch_model.safetensors"))
    cfg2, flat2 = P.load_unet_weights(str(d))
    assert cfg2 == cfg
    assert torch.equal(flat2, flat)
    table, _ = unet_spec.param_offsets(cfg)
    off, shape = table["down_blocks_0/attentions_0/proj_in/kernel"]
    hwio = sd["down_blocks.0.attentions.0.proj_in.weight"].permute(2, 3, 1, 0)
    assert torch.equal(flat2[off:off + hwio.numel()].view(shape), hwio)
