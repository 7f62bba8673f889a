"""The grouped time-embedding projection launch (one launch instead of one per ResNet block, bit-identical to the
separate launches) and the aesthetic reward model on the GPU kernels (CLIP ViT image
tower + LAION head against the oracle pinned to `transformers`)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("batch", [1, 2, 16, 40])
def test_dense_small_grouped_is_bit_identical(batch):
    from ddpo_b200 import ops
    g = torch.Generator().manual_seed(0)
    k, ns = 256, [64, 320, 96, 640]
    x = torch.randn(batch, k, generator=g).to(DEV)
    params, entries, off = [], [], 0
    for n in ns:
        w, b = torch.randn(k, n, generator=g) / 16, torch.randn(n, generator=g)
        entries.append((off, off + k * n, None, n))
        params += [w.reshape(-1), b]
        off += k * n + n
    flat = torch.cat(params).to(DEV)
    y_off, fixed = 0, []
    for (w_off, b_off, _, n) in entries:
        fixed.append((w_off, b_off, y_off, n))
        y_off += batch * n
    table, ctas = ops.dense_small_group_table(fixed, DEV)
    y_all = torch.zeros(y_off, device=DEV)
    ops.dense_small_grouped(x, flat, y_all, table, len(ns), ctas, batch, k)
    torch.cuda.synchronize()
    for (w_off, b_off, yo, n) in fixed:
        ref = torch.empty(batch, n, device=DEV)
        ops.dense_small(x, flat[w_off:w_off + k * n].view(k, n), flat[b_off:b_off + n], ref, batch, k, n)
        torch.cuda.synchronize()
        assert torch.equal(y_all[yo:yo + batch * n].view(batch, n), ref)


@pytest.mark.parametrize("cfg_name,batch", [("TINY", 2), ("SMALL", 4)])
def test_unet_grouped_temb_matches_separate_launches(cfg_name, batch):
    """Each of the 22 projections the U-Net's grouped launch wrote (at its real parameter-table offsets) equals a separate
    dense_small launch on that block's own time_emb_proj parameters and the same silu(temb)"""
    from ddpo_b200 import ops, unet_spec
    from ddpo_b200.unet import UNet
    cfg = getattr(unet_spec, cfg_name)
    flat = unet_spec.init_flat_params(cfg, 0)
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(batch, 4, cfg.sample_size, cfg.sample_size, generator=g).to(DEV)
    ctx = torch.randn(batch, cfg.ctx_len, cfg.cross_attention_dim, generator=g).to(DEV)
    ts = torch.tensor([981, 441, 21, 1][:batch], dtype=torch.int32, device=DEV)
    net = UNet(cfg, flat, DEV)
    net.prepare_context(ctx)
    net.enable_training()
    tape = []
    net.forward(lat, ts, tape=tape)    # with a tape the arena keeps temb_act and the grouped output alive
    temb_act = next(d for kind, d in tape if kind == "head")["temb_act"]
    te = temb_act.shape[1]
    assert len(net._tproj_views) == 22
    for name, got in net._tproj_views.items():
        w, bias = net.p(name + "/time_emb_proj/kernel"), net.p(name + "/time_emb_proj/bias")
        n = w.shape[1]
        ref = torch.empty(batch, n, device=DEV)
        ops.dense_small(temb_act, w, bias, ref, batch, te, n)
        torch.cuda.synchronize()
        assert torch.equal(got, ref), name


# ------------------------------------------------------------------ aesthetic reward model (clip_vision.py) ----
def test_vision_kernels():
    from ddpo_b200 import ops
    g = torch.Generator().manual_seed(0)
    img = torch.randn(2, 56, 56, 3, generator=g).to(DEV)
    out = torch.empty(2 * 16, 640, dtype=torch.bfloat16, device=DEV)
    ops.patchify_bf16(img, out, 14)
    ref = img.reshape(2, 4, 14, 4, 14, 3).permute(0, 1, 3, 2, 4, 5).reshape(32, 588)
    torch.cuda.synchronize()
    assert torch.equal(out[:, :588], ref.to(torch.bfloat16)) and float(out[:, 588:].abs().max()) == 0.0
    pe, cls, pos = torch.randn(32, 128, generator=g).to(DEV), torch.randn(128, generator=g).to(DEV), torch.randn(17, 128, generator=g).to(DEV)
    tok = torch.empty(2 * 17, 128, device=DEV)
    ops.vit_tokens(pe, cls, pos, tok, 2, 16, 128)
    want = torch.cat([cls.expand(2, 1, 128), pe.view(2, 16, 128)], 1) + pos[None]
    torch.cuda.synchronize()
    assert torch.equal(tok.view(2, 17, 128), want)
    x = torch.randn(5, 768, generator=g).to(DEV)
    y = torch.empty_like(x)
    ops.l2norm_rows(x, y)
    torch.cuda.synchronize()
    np.testing.assert_allclose(y.cpu().numpy(), (x / x.norm(dim=-1, keepdim=True)).cpu().numpy(), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("b", [3, 8])
def test_aesthetic_scorer_matches_oracle(b):
    from ddpo_b200 import clip_vision as CV
    from oracle import clip_vision as OCV
    cfg = CV.VIT_TINY
    flat = CV.init_flat_params(cfg, 0)
    sc = CV.AestheticScorer(cfg, flat, DEV)
    x = torch.randn(b, cfg.image_size, cfg.image_size, 3, generator=torch.Generator().manual_seed(2))
    feats = sc.image_features(x)
    scores = sc.score_features(feats)
    torch.cuda.synchronize()
    ref = OCV.image_features(CV.views(flat, cfg), cfg, x)
    rel = ((feats.cpu() - ref).norm() / ref.norm()).item()
    assert rel < 2e-2, rel
    np.testing.assert_allclose(scores.cpu().numpy(), OCV.aesthetic_score(CV.views(flat, cfg), ref).numpy(), rtol=5e-2, atol=5e-3)
    alone = sc.image_features(x[1:2])
    torch.cuda.synchronize()
    assert torch.equal(alone[0], feats[1])                       # batch invariant


def test_aesthetic_scorer_full_size_runs():
    from ddpo_b200 import clip_vision as CV
    sc = CV.AestheticScorer(CV.VIT_L14, device=DEV, seed=0)
    imgs = np.random.default_rng(0).random((8, 512, 512, 3)).astype(np.float32)
    s = sc(imgs, chunk=8)
    assert s.shape == (8, 1) and np.isfinite(s).all()
