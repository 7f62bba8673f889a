"""VAE decoder (ddpo_b200/vae.py + csrc/vae.cu, igemm rows wider than a tile) and the trajectory row gather vs
plain PyTorch fp32 references and the CPU oracle (oracle/vae.py)."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _setup():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def bf(x):
    return x.to(torch.bfloat16)


def _prep_w(w_kn):
    from ddpo_b200 import ops
    k, n = w_kn.shape
    dst = torch.empty(n, k, dtype=torch.bfloat16, device=DEV)
    ops.prep_weight(w_kn.contiguous(), dst, k, n)
    return dst


@pytest.mark.parametrize("rows,n,scale", [(4, 64, 0.125), (64, 1024, 1 / math.sqrt(128)), (33, 4096, 1 / math.sqrt(512))])
def test_softmax_rows(rows, n, scale):
    from ddpo_b200 import ops
    g = torch.Generator().manual_seed(0)
    s = (torch.randn(rows, n, generator=g) * 30).to(DEV)
    p = torch.empty(rows, n, dtype=torch.bfloat16, device=DEV)
    ops.softmax_rows(s, p, scale)
    torch.cuda.synchronize()
    ref = torch.softmax(s * scale, dim=-1)
    assert (p.float() - ref).abs().max().item() < 4e-3 * ref.max().item() + 1e-6
    np.testing.assert_allclose(p.float().sum(-1).cpu().numpy(), 1.0, atol=2e-2)


def test_post_quant_and_conv_out():
    from ddpo_b200 import ops
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(3, 4, 16, 8, generator=g).to(DEV)
    w = torch.randn(4, 4, generator=g).to(DEV)
    bias = torch.randn(4, generator=g).to(DEV)
    out = torch.empty_like(lat)
    ops.vae_post_quant(lat, w, bias, out, scaling=0.18215)
    ref = torch.einsum("bihw,io->bohw", lat / 0.18215, w) + bias[None, :, None, None]
    torch.cuda.synchronize()
    np.testing.assert_allclose(out.cpu().numpy(), ref.cpu().numpy(), rtol=1e-5, atol=1e-5)
    b, h, wd, cin = 2, 16, 32, 64
    x = torch.randn(b, h, wd, cin, generator=g).to(DEV)
    wk = (torch.randn(3, 3, cin, 3, generator=g) / math.sqrt(9 * cin)).to(DEV)
    bo = torch.randn(3, generator=g).to(DEV)
    raw = torch.empty(b, 3, h, wd, device=DEV)
    img = torch.empty(b, h, wd, 3, device=DEV)
    ops.vae_conv_out(x, wk, bo, b, h, wd, cin, raw_nchw=raw, img_nhwc=img)
    torch.cuda.synchronize()
    rr = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), wk.permute(3, 2, 0, 1), bo, padding=1)
    np.testing.assert_allclose(raw.cpu().numpy(), rr.cpu().numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(img.cpu().numpy(), (rr / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1).cpu().numpy(),
                               rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("b,h,w,c,n,ks", [(1, 4, 256, 64, 64, 3), (2, 256, 256, 64, 64, 3), (1, 8, 512, 64, 128, 3),
                                          (1, 4, 256, 128, 64, 1), (1, 8, 256, 64, 64, 3), (2, 2, 1024, 64, 64, 3)])
def test_igemm_conv_rows_wider_than_a_tile(b, h, w, c, n, ks):
    """W > 128: a pixel row spans W/128 tiles; left/right zero padding must come from the TMA box at x = -1 / W"""
    from ddpo_b200 import ops
    g = torch.Generator().manual_seed(2)
    x = bf(torch.randn(b, h, w, c, generator=g)).to(DEV)
    wk = (torch.randn(ks, ks, c, n, generator=g) / math.sqrt(ks * ks * c)).to(DEV)
    bias = torch.randn(n, generator=g).to(DEV)
    res = torch.randn(b * h * w, n, generator=g).to(DEV)
    out = torch.zeros(b * h * w, n, device=DEV)
    ops.igemm(a0=x, wt=_prep_w(wk.reshape(ks * ks * c, n)), n=n, c0=c, conv=(b, h, w), taps=ks * ks, bias=bias,
              residual=res, out_f32=out)
    torch.cuda.synchronize()
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), bf(wk).float().permute(3, 2, 0, 1), bias,
                                     padding=ks // 2).permute(0, 2, 3, 1).reshape(b * h * w, n) + res
    err = (out - ref).abs().max().item()
    assert err < 2e-3 * max(1.0, ref.abs().max().item()), f"max err {err}"


def test_gather_rows():
    from ddpo_b200 import ops
    g = torch.Generator().manual_seed(3)
    src = torch.randn(51 * 7, 4 * 16 * 16, generator=g).to(DEV)
    idx = torch.randint(0, src.shape[0], (40,), generator=g)
    dst = torch.empty(40, src.shape[1], device=DEV)
    ops.gather_rows(src, idx.to(DEV), dst)
    torch.cuda.synchronize()
    assert torch.equal(dst.cpu(), src.cpu()[idx])


def _decode_both(cfg_name, b, seed=0, decode_batch=2):
    from ddpo_b200 import vae as V
    from oracle import vae as OV
    cfg = getattr(V, cfg_name)
    flat = V.init_flat_params(cfg, seed)
    lat = torch.randn(b, 4, cfg.sample_size, cfg.sample_size, generator=torch.Generator().manual_seed(seed + 5)) * 0.18215
    dec = V.VAEDecoder(cfg, flat, DEV, decode_batch=decode_batch)
    img, raw = dec.decode(lat.to(DEV), want_raw=True, want_images=True)
    torch.cuda.synchronize()
    img_r, raw_r = OV.decode(V.views(flat, cfg), cfg, lat)
    return img.cpu(), raw.cpu(), img_r, raw_r


@pytest.mark.parametrize("cfg_name,b,decode_batch", [("VAE_MICRO", 2, 2), ("VAE_MICRO", 3, 2), ("VAE_TINY", 2, 1)])
def test_vae_decode_matches_oracle(cfg_name, b, decode_batch):
    img, raw, img_r, raw_r = _decode_both(cfg_name, b, decode_batch=decode_batch)
    assert img.shape == img_r.shape and raw.shape == raw_r.shape
    rel = ((raw - raw_r).norm() / raw_r.norm()).item()
    assert rel < 3e-2, f"decoder output relative L2 error {rel}"       # bf16 operands through ~30 layers
    assert (img - img_r).abs().max().item() < 0.1
    assert float(img.min()) >= 0.0 and float(img.max()) <= 1.0


def test_vae_decode_is_batch_invariant():
    """an image decodes to the same bits alone or inside a batch (fixed reduction orders, per-sample GroupNorm)"""
    from ddpo_b200 import vae as V
    cfg = V.VAE_MICRO
    dec = V.VAEDecoder(cfg, V.init_flat_params(cfg, 0), DEV, decode_batch=4)
    lat = (torch.randn(4, 4, 8, 8, generator=torch.Generator().manual_seed(1)) * 0.18215).to(DEV)
    a = dec.decode(lat)
    b = dec.decode(lat[2:3])
    torch.cuda.synchronize()
    assert torch.equal(a[2:3], b)


def test_vae_decode_full_size_properties():
    """SD decoder at 64x64 latents -> 512x512: shape, range, finite, and agreement of two identical latents"""
    from ddpo_b200 import vae as V
    dec = V.VAEDecoder(V.SD_VAE, device=DEV, seed=3, decode_batch=2)
    lat = torch.randn(1, 4, 64, 64, generator=torch.Generator().manual_seed(2)).mul(0.18215).expand(2, -1, -1, -1)
    img = dec.decode(lat.contiguous().to(DEV))
    torch.cuda.synchronize()
    assert img.shape == (2, 512, 512, 3) and torch.isfinite(img).all()
    assert float(img.min()) >= 0.0 and float(img.max()) <= 1.0 and float(img.std()) > 1e-3
    assert torch.equal(img[0], img[1])


# ------------------------------------------------------------------------------------------ VAE encoder ----
@pytest.mark.parametrize("b,h,w,c,n", [(2, 8, 8, 64, 64), (1, 64, 64, 128, 128), (2, 128, 128, 64, 64), (1, 256, 256, 128, 128)])
def test_igemm_stride2_without_low_padding(b, h, w, c, n):
    """the VAE encoder's down-sample: Flax pad ((0,1),(0,1)) + VALID 3x3 stride 2 == out[y,x] = sum in[2y+dy, 2x+dx];
    (h, w) is the OUTPUT grid; output rows up to 256 pixels wide (two 128-pixel tiles per row, 256-element TMA boxes)."""
    from ddpo_b200 import ops
    g = torch.Generator().manual_seed(30)
    x = torch.randn(b, 2 * h, 2 * w, c, generator=g).to(torch.bfloat16).to(DEV)
    wt = (torch.randn(3, 3, c, n, generator=g) / (3 * c ** 0.5)).to(DEV)
    bias = torch.randn(n, generator=g).to(DEV)
    wb = torch.empty(n, 9 * c, dtype=torch.bfloat16, device=DEV)
    ops.prep_weight(wt.reshape(9 * c, n).contiguous(), wb, 9 * c, n)
    out = torch.zeros(b * h * w, n, device=DEV)
    ops.igemm(a0=x, wt=wb, n=n, c0=c, conv=(b, h, w), taps=9, stride=2, no_low_pad=True, bias=bias, out_f32=out)
    torch.cuda.synchronize()
    xin = torch.nn.functional.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1))
    ref = torch.nn.functional.conv2d(xin, wt.to(torch.bfloat16).float().permute(3, 2, 0, 1), bias, stride=2)
    ref = ref.permute(0, 2, 3, 1).reshape(b * h * w, n)
    assert (out - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())


def test_vae_encoder_kernels():
    from ddpo_b200 import ops
    g = torch.Generator().manual_seed(31)
    img = torch.rand(2, 24, 40, 3, generator=g).to(DEV)
    out = torch.empty(2, 3, 24, 40, device=DEV)
    ops.vae_image_to_nchw(img, out)
    assert torch.equal(out, ((img - 0.5) / 0.5).permute(0, 3, 1, 2).contiguous())
    b, h, w, c = 2, 16, 8, 128
    x = torch.randn(b, h, w, c, generator=g).to(DEV)
    wk = (torch.randn(3, 3, c, 8, generator=g) / 30).to(DEV)
    bias = torch.randn(8, generator=g).to(DEV)
    wq = torch.randn(1, 1, 8, 8, generator=g).to(DEV) * 20      # large: both logvar clip bounds are exercised
    bq = torch.randn(8, generator=g).to(DEV)
    mom = torch.empty(b, h, w, 8, device=DEV)
    ops.vae_encoder_head(x, wk, bias, wq, bq, mom, b, h, w, c)
    torch.cuda.synchronize()
    hcv = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), wk.permute(3, 2, 0, 1), bias, padding=1)
    m = torch.einsum("bihw,io->bhwo", hcv, wq.reshape(8, 8)) + bq
    ref = torch.cat([m[..., :4], m[..., 4:].clamp(-30.0, 20.0)], -1)
    assert (mom - ref).abs().max().item() < 1e-3 * max(1.0, ref.abs().max().item())
    assert float(mom[..., 4:].max()) == 20.0 and float(mom[..., 4:].min()) == -30.0


@pytest.mark.parametrize("cfg_name,b,px", [("VAE_MICRO", 3, 64), ("VAE_TINY", 2, 256)])
def test_vae_encode_matches_oracle(cfg_name, b, px):
    from ddpo_b200 import vae as V
    from oracle import vae as OV
    cfg = getattr(V, cfg_name)
    flat = V.init_flat_params(cfg, 2, part="encoder")
    enc = V.VAEEncoder(cfg, flat, device=DEV, decode_batch=2)
    img = torch.rand(b, px, px, 3, generator=torch.Generator().manual_seed(9))
    mom = enc.encode(img)
    torch.cuda.synchronize()
    ref = OV.encode(V.views(flat, cfg, part="encoder"), cfg, img)
    assert tuple(mom.shape) == tuple(ref.shape) == (b, px // 8, px // 8, 8)
    rel = ((mom.cpu() - ref).norm() / ref.norm()).item()
    assert rel < 3e-2, rel
    alone = enc.encode(img[1:2])
    torch.cuda.synchronize()
    assert torch.equal(alone[0], mom[1])        # batch invariant


def test_vae_encode_full_size_and_callback():
    """SD VAE encoder at 512 px (first down-sample writes rows 256 pixels wide) through the `vae` callback of the RWR path."""
    from ddpo_b200 import vae as V
    from ddpo_b200.training import callbacks as C
    from oracle import vae as OV
    enc = V.VAEEncoder(V.SD_VAE, device=DEV, seed=4, decode_batch=1)
    img = np.random.default_rng(0).random((2, 512, 512, 3)).astype(np.float32)
    mom, info = C.callback_fns["vae"](encoder=enc)(img)
    assert mom.shape == (2, 64, 64, 8) and np.isfinite(mom).all() and mom[..., 4:].max() <= 20.0 and mom[..., 4:].min() >= -30.0
    ref = OV.encode(V.views(enc.params.cpu(), V.SD_VAE, part="encoder"), V.SD_VAE, torch.from_numpy(img[:1])).numpy()
    rel = np.linalg.norm(mom[:1] - ref) / np.linalg.norm(ref)
    assert rel < 3e-2, rel


def test_image_to_uint8_matches_the_reference_cast():
    """device-side `(image * 255).astype(np.uint8)` (reference callbacks.py:181): bit-exact incl. 0, 1 and values a hair below k/255"""
    from ddpo_b200 import ops
    rng = np.random.default_rng(3)
    x = rng.random((2, 64, 48, 3)).astype(np.float32)
    x.reshape(-1)[:8] = [0.0, 1.0, 0.5, 254.999 / 255, 255 / 255, 1 / 255, np.nextafter(np.float32(2 / 255), np.float32(0)), 0.99999994]
    d = torch.from_numpy(x).to(DEV)
    u8 = torch.empty(x.shape, dtype=torch.uint8, device=DEV)
    ops.image_to_uint8(d, u8)
    torch.cuda.synchronize()
    assert np.array_equal(u8.cpu().numpy(), (x * 255).astype(np.uint8))
