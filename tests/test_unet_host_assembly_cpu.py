"""The U-Net's HOST assembly (ddpo_b200/unet.py: kernel sequencing of the sampling forward, weight preparation incl. the
GEGLU tile interleave, two-source norms / convolutions, cross-attention K/V cache, skip bookkeeping) dry-run on the
torch-CPU emulation of the ops it calls (tests/_cpu_ops_emulator.py) against the oracle -- and the grouped
time-embedding launch against per-block launches.  The CUDA kernels themselves are checked on the GPU box."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))


def _net(monkeypatch, cfg, flat):
    import _cpu_ops_emulator as E
    from ddpo_b200 import unet as U
    monkeypatch.setattr(U, "ops", E)
    monkeypatch.setattr(U, "Arena", E.CpuArena)
    return U.UNet(cfg, flat, device="cpu")


@pytest.mark.parametrize("batch,scalar_t", [(2, False), (3, True)])
def test_unet_forward_host_assembly_matches_oracle(monkeypatch, batch, scalar_t):
    from ddpo_b200 import unet_spec
    from oracle.unet import UNetOracle
    cfg = unet_spec.TINY
    flat = unet_spec.init_flat_params(cfg, 0)
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(batch, 4, cfg.sample_size, cfg.sample_size, generator=g)
    ctx = torch.randn(batch, cfg.ctx_len, cfg.cross_attention_dim, generator=g)
    ts = torch.tensor([981] if scalar_t else [981, 21, 441][:batch], dtype=torch.int32)
    net = _net(monkeypatch, cfg, flat)
    net.prepare_context(ctx)
    eps = net.forward(lat, ts)
    with torch.no_grad():
        ref = UNetOracle(cfg, unet_spec.views(flat, cfg))(lat, ts.expand(batch).long() if scalar_t else ts.long(), ctx)
    rel = ((eps - ref).norm() / ref.norm()).item()
    assert eps.shape == ref.shape and rel < 2e-2, rel            # bf16 operands through ~60 layers (GPU: 1.0e-2)
    # a second call with another context must not see the first one's K/V (persistent buffers are refilled)
    ctx2 = torch.randn(batch, cfg.ctx_len, cfg.cross_attention_dim, generator=g)
    net.prepare_context(ctx2)
    eps2 = net.forward(lat, ts)
    assert not torch.equal(eps2, eps)
    net.prepare_context(ctx)
    assert torch.equal(net.forward(lat, ts), eps)


def test_grouped_time_embedding_matches_per_block_dense_small(monkeypatch):
    """each block's projection from the grouped launch (at the U-Net's parameter-table offsets) equals a separate
    dense_small on that block's own time_emb_proj parameters"""
    import _cpu_ops_emulator as E
    from ddpo_b200 import unet_spec
    cfg = unet_spec.TINY
    flat = unet_spec.init_flat_params(cfg, 0)
    g = torch.Generator().manual_seed(2)
    lat = torch.randn(2, 4, cfg.sample_size, cfg.sample_size, generator=g)
    ctx = torch.randn(2, cfg.ctx_len, cfg.cross_attention_dim, generator=g)
    ts = torch.tensor([500, 3], dtype=torch.int32)
    net = _net(monkeypatch, cfg, flat)
    net.enable_training()
    net.prepare_context(ctx)
    tape = []
    net.forward(lat, ts, tape=tape)
    temb_act = next(d for kind, d in tape if kind == "head")["temb_act"]
    assert len(net._temb_names) == 22 and sorted(net._tproj_views) == sorted(net._temb_names)
    for name, got in net._tproj_views.items():
        w, bias = net.p(name + "/time_emb_proj/kernel"), net.p(name + "/time_emb_proj/bias")
        ref = torch.empty(2, w.shape[1])
        E.dense_small(temb_act, w, bias, ref, 2, w.shape[0], w.shape[1])
        assert torch.equal(got, ref), name
    tab = net._temb_tables[2]
    assert tab[1] == sum((n + 31) // 32 for _, _, n in tab[2])       # CTA count of the grouped launch


@pytest.mark.parametrize("batch", [2])
def test_unet_backward_host_assembly_matches_oracle_autograd(monkeypatch, batch):
    """the taped forward + hand-written backward sequencing of ddpo_b200/unet.py (gradient routing through skips /
    two-source layers, bias / time-embedding / norm / attention / GEGLU gradients, accumulation into the flat buffer),
    dry-run on the ops emulator against torch autograd through the oracle"""
    from ddpo_b200 import unet_spec
    from oracle.unet import UNetOracle
    cfg = unet_spec.TINY
    flat = unet_spec.init_flat_params(cfg, 0)
    g = torch.Generator().manual_seed(11)
    s = cfg.sample_size
    lat = torch.randn(batch, 4, s, s, generator=g)
    ctx = torch.randn(batch, cfg.ctx_len, cfg.cross_attention_dim, generator=g)
    ts = torch.tensor([981, 21][:batch], dtype=torch.int32)
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
    # accumulation semantics: a second pass doubles the gradient buffer
    first = net.grads.clone()
    tape = []
    net.forward(lat, ts, tape=tape)
    net.backward(tape, d_eps)
    np.testing.assert_allclose(net.grads.numpy(), 2 * first.numpy(), rtol=1e-4, atol=1e-7)
