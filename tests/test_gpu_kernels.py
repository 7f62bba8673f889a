"""GPU parity tests of the individual CUDA kernels (through the C ABI) against plain
PyTorch fp32 references and the CPU oracle.  Run on an H100: ``pytest -m gpu``."""
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
    from ddpo_b200 import _lib
    assert _lib.lib().ddpo_device_sm_count() > 0
    yield


def bf(x):
    return x.to(torch.bfloat16)


def rel_err(a, b):
    a = a.float()
    b = b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


# ----------------------------------------------------------------------- PRNG ----
@pytest.mark.parametrize("n", [2, 7, 4096, 2 * 4 * 64 * 64 + 3])
def test_threefry_normal_matches_oracle(n):
    from ddpo_b200 import ops
    from oracle import threefry
    key = (0x9E3779B9, 12345)
    kd = ops.key_tensor([key], DEV)
    out = torch.empty(n, device=DEV)
    ops.threefry_normal(kd, out)
    ref = threefry.normal(np.array(key, np.uint32), (n,))
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=0, atol=2e-6)


def test_threefry_host_split_matches_oracle():
    from ddpo_b200 import ops
    from oracle import threefry
    k = ops.prng_key(0)
    assert k == (0, 0)
    s = ops.threefry_split(k, 2)
    assert s == [(4146024105, 967050713), (2718843009, 1272950319)]  # published JAX values
    s5 = ops.threefry_split((123, 456), 5)
    ref = threefry.split(np.array([123, 456], np.uint32), 5)
    assert [tuple(int(v) for v in r) for r in ref] == s5


# ----------------------------------------------------------------------- DDIM ----
def _sched():
    from oracle import scheduler as S
    st = S.set_timesteps(S.SD_CONFIG, S.create_state(S.SD_CONFIG), 50)
    return S, st


@pytest.mark.parametrize("batch,t_scalar", [(2, True), (3, True), (4, False)])
def test_ddim_step_sample_and_score(batch, t_scalar):
    from ddpo_b200 import ops
    from oracle import threefry
    from oracle.ppo import cfg_combine
    S, st = _sched()
    n = 4 * 16 * 16
    rng = np.random.default_rng(0)
    eu = rng.standard_normal((batch, n)).astype(np.float32)
    ec = rng.standard_normal((batch, n)).astype(np.float32)
    x = rng.standard_normal((batch, n)).astype(np.float32)
    ts = np.array([981] if t_scalar else [981, 21, 1, 501][:batch], np.int32)
    key = (7, 9)
    g, eta = 5.0, 1.0
    ac = torch.tensor(st.alphas_cumprod, device=DEV)
    ws = ops.ddim_workspace(batch, DEV)
    prev = torch.empty(batch, n, device=DEV)
    lp = torch.empty(batch, device=DEV)
    teu, tec, tx = (torch.tensor(a, device=DEV) for a in (eu, ec, x))
    tts = torch.tensor(ts, device=DEV)
    ops.ddim_step_sample(teu, tec, tx, ac, tts, float(st.final_alpha_cumprod), 20, g, eta, ops.key_tensor([key], DEV),
                         prev, lp, ws)
    eps = cfg_combine(eu, ec, g)
    tt = int(ts[0]) if t_scalar else ts
    rprev, _, rlp = S.step(S.SD_CONFIG, st, eps, tt, x, key=np.array(key, np.uint32), eta=eta)
    np.testing.assert_allclose(prev.cpu().numpy(), rprev, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(lp.cpu().numpy(), rlp, rtol=1e-5, atol=1e-5)
    # score mode on the produced sample returns the same log-prob (bit-reproducible reduction)
    lp2 = torch.empty(batch, device=DEV)
    ops.ddim_logprob_fwd(teu, tec, tx, prev, ac, tts, float(st.final_alpha_cumprod), 20, g, eta, lp2, ws)
    _, _, rlp2 = S.step(S.SD_CONFIG, st, eps, tt if not t_scalar else np.full(batch, tt), x,
                        prev_sample=prev.cpu().numpy(), eta=eta)
    np.testing.assert_allclose(lp2.cpu().numpy(), rlp2, rtol=1e-5, atol=1e-5)
    assert torch.equal(lp, lp2), "sample-mode and score-mode log-probs must be bit identical"
    # backward
    dl = torch.tensor(rng.standard_normal(batch).astype(np.float32), device=DEV)
    du = torch.empty(batch, n, device=DEV)
    dc = torch.empty(batch, n, device=DEV)
    ops.ddim_logprob_bwd(teu, tec, tx, prev, ac, tts, float(st.final_alpha_cumprod), 20, g, eta, dl, du, dc, ws)
    gref = S.logprob_grad_eps(S.SD_CONFIG, st, eps, tt if not t_scalar else np.full(batch, tt), x,
                              prev.cpu().numpy(), eta, dl.cpu().numpy())
    np.testing.assert_allclose(dc.cpu().numpy(), g * gref, rtol=2e-4, atol=1e-7)
    np.testing.assert_allclose(du.cpu().numpy(), (1 - g) * gref, rtol=2e-4, atol=1e-7)


@pytest.mark.parametrize("pred", ["sample", "v_prediction"])
def test_ddim_prediction_types(pred):
    """The `sample` and `v_prediction` branches of FlaxDDIMScheduler.step (scheduling_ddim_flax.py:307-316): sample
    mode, score mode and the backward against the oracle; sample-mode and score-mode log-probs bit identical."""
    from dataclasses import replace
    from ddpo_b200 import ops
    from oracle.ppo import cfg_combine
    S, st = _sched()
    cfg = replace(S.SD_CONFIG, prediction_type=pred)
    batch, n = 3, 4 * 16 * 16
    rng = np.random.default_rng(3)
    eu, ec, x = (rng.standard_normal((batch, n)).astype(np.float32) for _ in range(3))
    ts = np.array([981, 21, 501], np.int32)
    key, g, eta = (5, 11), 3.0, 1.0
    ac = torch.tensor(st.alphas_cumprod, device=DEV)
    ws = ops.ddim_workspace(batch, DEV)
    prev, lp, lp2 = torch.empty(batch, n, device=DEV), torch.empty(batch, device=DEV), torch.empty(batch, device=DEV)
    teu, tec, tx, tts = (torch.tensor(a, device=DEV) for a in (eu, ec, x, ts))
    fa = float(st.final_alpha_cumprod)
    ops.ddim_step_sample(teu, tec, tx, ac, tts, fa, 20, g, eta, ops.key_tensor([key], DEV), prev, lp, ws, pred=pred)
    m = cfg_combine(eu, ec, g)
    rprev, _, rlp = S.step(cfg, st, m, ts, x, key=np.array(key, np.uint32), eta=eta)
    np.testing.assert_allclose(prev.cpu().numpy(), rprev, rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(lp.cpu().numpy(), rlp, rtol=1e-5, atol=1e-5)
    ops.ddim_logprob_fwd(teu, tec, tx, prev, ac, tts, fa, 20, g, eta, lp2, ws, pred=pred)
    assert torch.equal(lp, lp2)
    # score mode on an unrelated next sample
    other = torch.tensor(rng.standard_normal((batch, n)).astype(np.float32), device=DEV)
    ops.ddim_logprob_fwd(teu, tec, tx, other, ac, tts, fa, 20, g, eta, lp2, ws, pred=pred)
    _, _, rlp2 = S.step(cfg, st, m, ts, x, prev_sample=other.cpu().numpy(), eta=eta)
    np.testing.assert_allclose(lp2.cpu().numpy(), rlp2, rtol=2e-5)
    dl = torch.tensor(rng.standard_normal(batch).astype(np.float32), device=DEV)
    du, dc = torch.empty(batch, n, device=DEV), torch.empty(batch, n, device=DEV)
    ops.ddim_logprob_bwd(teu, tec, tx, other, ac, tts, fa, 20, g, eta, dl, du, dc, ws, pred=pred)
    gref = S.logprob_grad_eps(cfg, st, m, ts, x, other.cpu().numpy(), eta, dl.cpu().numpy())
    np.testing.assert_allclose(dc.cpu().numpy(), g * gref, rtol=3e-4, atol=1e-6)
    np.testing.assert_allclose(du.cpu().numpy(), (1 - g) * gref, rtol=3e-4, atol=1e-6)
    with pytest.raises(ValueError):
        ops.ddim_logprob_fwd(teu, tec, tx, other, ac, tts, fa, 20, g, eta, lp2, ws, pred="velocity")


def test_ppo_loss_matches_oracle():
    from ddpo_b200 import ops
    from oracle import ppo
    rng = np.random.default_rng(1)
    n = 16
    old = rng.standard_normal(n).astype(np.float32)
    lp = (old + 3e-4 * rng.standard_normal(n)).astype(np.float32)
    lp[:4] = old[:4]
    adv = (20 * rng.standard_normal(n)).astype(np.float32)
    info = torch.empty(3, device=DEV)
    dl = torch.empty(n, device=DEV)
    ops.ppo_loss(torch.tensor(lp, device=DEV), torch.tensor(old, device=DEV), torch.tensor(adv, device=DEV), 1e-4, info,
                 dl)
    loss, rinfo, rdl = ppo.ppo_loss(lp, old, adv, 1e-4)
    np.testing.assert_allclose(info.cpu().numpy(), [rinfo["approx_kl"], rinfo["clipfrac"], rinfo["loss"]], rtol=1e-5,
                               atol=1e-9)
    np.testing.assert_allclose(dl.cpu().numpy(), rdl, rtol=1e-5, atol=1e-9)


# ----------------------------------------------------------------------- GEMM ----
def _prep_w(w_kn):
    """fp32 [K, N] -> bf16 [N, K] through the library's own prep kernel."""
    from ddpo_b200 import ops
    k, n = w_kn.shape
    dst = torch.empty(n, k, dtype=torch.bfloat16, device=DEV)
    ops.prep_weight(w_kn.contiguous(), dst, k, n)
    return dst


@pytest.mark.parametrize("m,k,n,bn", [(128, 64, 64, 0), (256, 128, 128, 0), (300, 320, 320, 0), (1000, 640, 1920, 0),
                                      (4096, 1280, 1280, 256), (77 * 2, 1024, 640, 0), (128, 64, 256, 64)])
def test_igemm_linear(m, k, n, bn):
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(0)
    a = torch.randn(m, k, generator=g).to(DEV)
    w = (torch.randn(k, n, generator=g) / math.sqrt(k)).to(DEV)
    bias = torch.randn(n, generator=g).to(DEV)
    res = torch.randn(m, n, generator=g).to(DEV)
    ab = bf(a).contiguous()
    wt = _prep_w(w)
    assert torch.equal(wt, bf(w).t().contiguous())
    out = torch.zeros(m, n, device=DEV)
    outb = torch.zeros(m, n, dtype=torch.bfloat16, device=DEV)
    ops.igemm(a0=ab, wt=wt, n=n, c0=k, m=m, bias=bias, residual=res, out_f32=out, out_bf16=outb, bn=bn)
    torch.cuda.synchronize()
    ref = ab.float() @ bf(w).float() + bias + res
    err = (out - ref).abs().max().item()
    assert err < 2e-3 * max(1.0, ref.abs().max().item()), f"max err {err}"
    assert rel_err(outb, ref) < 5e-3


def test_igemm_geglu():
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(1)
    m, c = 384, 128
    a = bf(torch.randn(m, c, generator=g)).to(DEV)
    w = (torch.randn(c, 8 * c, generator=g) / math.sqrt(c)).to(DEV)
    bias = torch.randn(8 * c, generator=g).to(DEV)
    wt = torch.empty(8 * c, c, dtype=torch.bfloat16, device=DEV)
    ops.prep_weight(w, wt, c, 8 * c, geglu_bn=256)
    bp = torch.empty_like(bias)
    ops.permute_geglu_bias(bias, bp, 8 * c, 256)
    out = torch.zeros(m, 4 * c, dtype=torch.bfloat16, device=DEV)
    ops.igemm(a0=a, wt=wt, n=8 * c, c0=c, m=m, bias=bp, out_bf16=out, geglu=True, bn=256)
    torch.cuda.synchronize()
    f = a.float() @ bf(w).float() + bias
    lin, gate = f.chunk(2, dim=-1)
    ref = lin * torch.nn.functional.gelu(gate, approximate="tanh")
    assert rel_err(out, ref) < 6e-3


def _widths(n):
    """Every tile width (the wgmma N of the implicit GEMM) that divides n."""
    return [w for w in (32, 64, 96, 128, 160, 192, 256) if n % w == 0]


def _geglu_natural(aux, n, bn):
    """Pre-activations stored tile-interleaved ([bn/2 linear | bn/2 gate] per tile) -> [linear | gate]."""
    m = aux.shape[0]
    return aux.view(m, n // bn, 2, bn // 2).permute(0, 2, 1, 3).reshape(m, n)


def _conv_ref(x_nhwc, w_hwio, bias, stride):
    y = torch.nn.functional.conv2d(x_nhwc.permute(0, 3, 1, 2), w_hwio.permute(3, 2, 0, 1), bias, stride=stride,
                                   padding=w_hwio.shape[0] // 2)
    return y.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("b,h,c0,c1,n,ks,stride", [
    (2, 8, 64, 0, 64, 3, 1), (1, 16, 128, 0, 128, 3, 1), (3, 8, 64, 0, 128, 3, 1), (2, 64, 64, 0, 64, 3, 1),
    (2, 32, 128, 64, 160, 3, 1), (2, 16, 64, 64, 64, 1, 1), (2, 16, 64, 0, 64, 3, 2), (2, 8, 128, 0, 64, 3, 2),
    (1, 4, 64, 0, 64, 3, 1), (5, 2, 64, 0, 64, 3, 1), (2, 64, 320, 0, 320, 3, 1)])
def test_igemm_conv(b, h, c0, c1, n, ks, stride):
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(2)
    hi = h * stride
    x0 = bf(torch.randn(b, hi, hi, c0, generator=g)).to(DEV)
    x1 = bf(torch.randn(b, hi, hi, c1, generator=g)).to(DEV) if c1 else None
    cin = c0 + c1
    w = (torch.randn(ks, ks, cin, n, generator=g) / math.sqrt(ks * ks * cin)).to(DEV)
    bias = torch.randn(n, generator=g).to(DEV)
    tvec = torch.randn(b, n, generator=g).to(DEV)
    wt = _prep_w(w.reshape(ks * ks * cin, n))
    out = torch.zeros(b * h * h, n, device=DEV)
    ops.igemm(a0=x0, a1=x1, wt=wt, n=n, c0=c0, c1=c1, conv=(b, h, h), taps=ks * ks, stride=stride, bias=bias,
              rowvec=tvec, rows_per_sample=h * h, rowvec_ld=n, out_f32=out)
    torch.cuda.synchronize()
    xin = x0.float() if x1 is None else torch.cat([x0.float(), x1.float()], dim=-1)
    ref = _conv_ref(xin, bf(w).float(), bias, stride) + tvec[:, None, None, :]
    ref = ref.reshape(b * h * h, n)
    err = (out - ref).abs().max().item()
    assert err < 2e-3 * max(1.0, ref.abs().max().item()), f"max err {err}"


def test_igemm_batch_invariance():
    """The same sample must produce bit-identical rows whatever the batch size / tile position."""
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(3)
    c, n, h = 128, 128, 8
    x = bf(torch.randn(6, h, h, c, generator=g)).to(DEV)
    w = (torch.randn(9 * c, n, generator=g) / math.sqrt(9 * c)).to(DEV)
    wt = _prep_w(w)
    big = torch.zeros(6 * h * h, n, device=DEV)
    ops.igemm(a0=x, wt=wt, n=n, c0=c, conv=(6, h, h), taps=9, out_f32=big)
    for i in (1, 4, 5):
        small = torch.zeros(h * h, n, device=DEV)
        ops.igemm(a0=x[i:i + 1].contiguous(), wt=wt, n=n, c0=c, conv=(1, h, h), taps=9, out_f32=small)
        assert torch.equal(small, big[i * h * h:(i + 1) * h * h])


# ------------------------------------------------------------------ attention ----
@pytest.mark.parametrize("b,heads,nq,nk", [(1, 1, 128, 128), (2, 2, 256, 256), (1, 1, 1024, 1024), (2, 5, 4096, 4096),
                                           (2, 2, 256, 77), (3, 4, 64, 64), (2, 2, 64, 77)])
def test_attention_fwd(b, heads, nq, nk):
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(4)
    c = heads * 64
    q = bf(torch.randn(b, nq, c, generator=g)).to(DEV)
    kv = bf(torch.randn(b, nk, 2 * c, generator=g)).to(DEV)
    out = torch.zeros(b, nq, c, dtype=torch.bfloat16, device=DEV)
    lse = torch.zeros(b, heads, nq, device=DEV)
    ops.attention_fwd(q, kv, kv[:, :, c:], out, b, heads, nq, nk, c, 2 * c, 2 * c, c, lse=lse)
    torch.cuda.synchronize()
    qh = q.float().view(b, nq, heads, 64).permute(0, 2, 1, 3)
    kh = kv[:, :, :c].float().reshape(b, nk, heads, 64).permute(0, 2, 1, 3)
    vh = kv[:, :, c:].float().reshape(b, nk, heads, 64).permute(0, 2, 1, 3)
    s = (qh @ kh.transpose(-1, -2)) * 0.125
    ref = (torch.softmax(s, dim=-1) @ vh).permute(0, 2, 1, 3).reshape(b, nq, c)
    assert rel_err(out, ref) < 1e-2
    assert (lse - torch.logsumexp(s, dim=-1)).abs().max().item() < 1e-3


@pytest.mark.parametrize("b,heads,nq,nk", [(2, 2, 256, 77), (3, 5, 4096, 77), (2, 20, 256, 77), (1, 2, 1024, 128), (2, 1, 384, 16),
                                           (2, 2, 300, 77)])
def test_cross_attention_is_batch_invariant(b, heads, nq, nk):
    """Cross-attention shapes (Nk <= 128, keys past nk masked inside one key block): every sample's output and LSE are
    bit-identical whether it is computed inside the batch or alone."""
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(41)
    c = heads * 64
    q = bf(torch.randn(b, nq, c, generator=g)).to(DEV)
    kv = bf(torch.randn(b, nk, 2 * c, generator=g)).to(DEV)
    outs = []
    for sl in (slice(0, b), slice(b - 1, b)):
        bb = sl.stop - sl.start
        qs, kvs = q[sl].contiguous(), kv[sl].contiguous()
        out = torch.zeros(bb, nq, c, dtype=torch.bfloat16, device=DEV)
        lse = torch.zeros(bb, heads, nq, device=DEV)
        ops.attention_fwd(qs, kvs, kvs[:, :, c:], out, bb, heads, nq, nk, c, 2 * c, 2 * c, c, lse=lse)
        torch.cuda.synchronize()
        outs.append((out, lse))
    assert torch.equal(outs[0][0][b - 1:], outs[1][0]) and torch.equal(outs[0][1][b - 1:], outs[1][1])
    outs.reverse()
    qh = q.float().view(b, nq, heads, 64).permute(0, 2, 1, 3)
    kh = kv[:, :, :c].float().reshape(b, nk, heads, 64).permute(0, 2, 1, 3)
    vh = kv[:, :, c:].float().reshape(b, nk, heads, 64).permute(0, 2, 1, 3)
    ref = (torch.softmax((qh @ kh.transpose(-1, -2)) * 0.125, dim=-1) @ vh).permute(0, 2, 1, 3).reshape(b, nq, c)
    assert rel_err(outs[1][0], ref) < 1e-2


# ---------------------------------------------------------------------- norms ----
@pytest.mark.parametrize("kind,b,h,c0,c1,n", [("conv", 20, 64, 320, 0, 320),      # 640 row tiles of 128 rows
                                              ("conv", 3, 32, 640, 320, 640),     # two-source K, two column tiles
                                              ("conv", 2, 16, 128, 0, 1280),      # 4 column tiles, 2 row tiles
                                              ("conv", 5, 8, 64, 0, 320),         # 320 rows: ragged last row tile
                                              ("lin", 1, 1000, 2048, 0, 960),     # ragged M, 3 column tiles, long K
                                              ("lin", 1, 70000, 256, 0, 320)])    # 547 row tiles, the last one ragged
def test_igemm_wide_tiles_bit_identical(kind, b, h, c0, c1, n):
    """The tile width is a scheduling choice: 160- and 32-column tiles give bit-identical outputs AND slab statistics."""
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(77)
    bias = torch.randn(n, generator=g).to(DEV)
    c = c0 + c1
    outs = []
    if kind == "conv":
        m = b * h * h
        x0 = bf(torch.randn(b, h, h, c0, generator=g)).to(DEV)
        x1 = bf(torch.randn(b, h, h, c1, generator=g)).to(DEV) if c1 else None
        w = (torch.randn(9 * c, n, generator=g) / math.sqrt(9 * c)).to(DEV)
        res = torch.randn(m, n, generator=g).to(DEV)
        tvec = torch.randn(b, n, generator=g).to(DEV)
        wb = _prep_w(w)
        for bn in (160, 32):
            out = torch.zeros(m, n, device=DEV)
            ob = torch.zeros(m, n, device=DEV, dtype=torch.bfloat16)
            st = torch.full(ops.gn_stats_shape(m, n), float("nan"), device=DEV)
            ops.igemm(a0=x0, a1=x1, wt=wb, n=n, c0=c0, c1=c1, conv=(b, h, h), taps=9, bias=bias, rowvec=tvec,
                      rows_per_sample=h * h, rowvec_ld=n, residual=res, out_f32=out, gn_stats=st, bn=bn)
            ops.igemm(a0=x0, a1=x1, wt=wb, n=n, c0=c0, c1=c1, conv=(b, h, h), taps=9, bias=bias, out_bf16=ob, bn=bn)
            outs.append((out, st, ob))
    else:
        m = h
        x = bf(torch.randn(m, c, generator=g)).to(DEV)
        w = (torch.randn(c, n, generator=g) / math.sqrt(c)).to(DEV)
        res = torch.randn(m, n, generator=g).to(DEV)
        wb = _prep_w(w)
        for bn in (160, 32):
            out = torch.zeros(m, n, device=DEV)
            ob = torch.zeros(m, n, device=DEV, dtype=torch.bfloat16)
            st = torch.full(ops.gn_stats_shape(m, n), float("nan"), device=DEV)
            ops.igemm(a0=x, wt=wb, n=n, c0=c, m=m, bias=bias, residual=res, out_f32=out, out_bf16=ob, gn_stats=st, bn=bn)
            outs.append((out, st, ob))
    torch.cuda.synchronize()
    ref = (x.float() @ bf(w).float() + bias + res) if kind == "lin" else None
    if ref is not None:
        assert (outs[0][0] - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())
    for a, bb in zip(outs[0], outs[1]):
        assert torch.isfinite(a.float()).all() and torch.equal(a, bb)


@pytest.mark.parametrize("b,hw,c0,c1,silu", [(2, 64, 64, 0, True), (2, 4096, 320, 0, True), (3, 1024, 1280, 640, True),
                                             (2, 256, 1280, 1280, False), (1, 16, 128, 64, True)])
def test_groupnorm_fwd(b, hw, c0, c1, silu):
    from ddpo_b200 import ops
    from oracle.unet import group_norm, silu as silu_ref
    g = torch.Generator(device="cpu").manual_seed(5)
    c = c0 + c1
    x0 = (torch.randn(b, hw, c0, generator=g) * 2 + 0.5).to(DEV)
    x1 = torch.randn(b, hw, c1, generator=g).to(DEV) if c1 else None
    sc = (1 + 0.1 * torch.randn(c, generator=g)).to(DEV)
    bi = (0.1 * torch.randn(c, generator=g)).to(DEV)
    ws = torch.zeros(ops.groupnorm_workspace_floats(b, hw, c), device=DEV)
    y = torch.zeros(b, hw, c, dtype=torch.bfloat16, device=DEV)
    yf = torch.zeros(b, hw, c, device=DEV)
    raw = torch.zeros(b, hw, c, dtype=torch.bfloat16, device=DEV)
    ops.groupnorm_fwd(x0, sc, bi, ws, b, hw, c0, x1=x1, c1=c1, silu=silu, y_bf16=y, y_f32=yf, raw_bf16=raw)
    torch.cuda.synchronize()
    x = x0 if x1 is None else torch.cat([x0, x1], dim=-1)
    ref = group_norm(x.view(b, hw, 1, c), sc, bi).view(b, hw, c)
    if silu:
        ref = silu_ref(ref)
    assert (yf - ref).abs().max().item() < 2e-4
    assert rel_err(y, ref) < 4e-3
    assert torch.equal(raw, bf(x))


def _slab_stats_ref(y):
    rows, n = y.shape
    pad = (-rows) % 32
    yp = torch.cat([y, y.new_zeros(pad, n)]) if pad else y
    t = yp.double().reshape(-1, 32, n)
    return torch.stack([t.sum(1), (t * t).sum(1)], -1).float()


@pytest.mark.parametrize("kind,b,h,c,n", [("conv", 2, 16, 128, 160), ("conv", 4, 32, 64, 320), ("conv", 3, 8, 128, 128),
                                          ("lin", 1, 1000, 128, 256), ("lin", 1, 333, 64, 96), ("lin", 1, 4096, 320, 320)])
def test_igemm_gn_slab_stats(kind, b, h, c, n):
    """The epilogue's per-(32-row slab, column) sums of what it writes (bias + row vector + residual included)."""
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(31)
    bias = torch.randn(n, generator=g).to(DEV)
    if kind == "conv":
        m = b * h * h
        x = bf(torch.randn(b, h, h, c, generator=g)).to(DEV)
        w = (torch.randn(9 * c, n, generator=g) / math.sqrt(9 * c)).to(DEV)
        res = torch.randn(m, n, generator=g).to(DEV)
        tvec = torch.randn(b, n, generator=g).to(DEV)
        out = torch.zeros(m, n, device=DEV)
        st = torch.full(ops.gn_stats_shape(m, n), float("nan"), device=DEV)
        ops.igemm(a0=x, wt=_prep_w(w), n=n, c0=c, conv=(b, h, h), taps=9, bias=bias, rowvec=tvec, rows_per_sample=h * h,
                  rowvec_ld=n, residual=res, out_f32=out, gn_stats=st)
        ref_out = torch.zeros(m, n, device=DEV)
        ops.igemm(a0=x, wt=_prep_w(w), n=n, c0=c, conv=(b, h, h), taps=9, bias=bias, rowvec=tvec, rows_per_sample=h * h,
                  rowvec_ld=n, residual=res, out_f32=ref_out)
    else:
        m = h
        x = bf(torch.randn(m, c, generator=g)).to(DEV)
        w = (torch.randn(c, n, generator=g) / math.sqrt(c)).to(DEV)
        res = torch.randn(m, n, generator=g).to(DEV)
        out = torch.zeros(m, n, device=DEV)
        st = torch.full(ops.gn_stats_shape(m, n), float("nan"), device=DEV)
        ops.igemm(a0=x, wt=_prep_w(w), n=n, c0=c, m=m, bias=bias, residual=res, out_f32=out, gn_stats=st)
        ref_out = torch.zeros(m, n, device=DEV)
        ops.igemm(a0=x, wt=_prep_w(w), n=n, c0=c, m=m, bias=bias, residual=res, out_f32=ref_out)
    torch.cuda.synchronize()
    assert torch.equal(out, ref_out), "asking for statistics must not change the output"
    ref = _slab_stats_ref(out)
    assert torch.isfinite(st).all()
    assert (st - ref).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("b,hw,c0,c1,silu", [(2, 64, 64, 0, True), (2, 4096, 320, 0, True), (3, 1024, 1280, 640, True),
                                             (2, 256, 1280, 1280, False), (16, 64, 1280, 1280, True), (2, 4096, 640, 320, True)])
def test_groupnorm_fwd_from_slab_stats(b, hw, c0, c1, silu):
    """One-pass GroupNorm: statistics from the producer's slab sums (here written by torch); the result agrees with the
    oracle and with the two-pass path."""
    from ddpo_b200 import ops
    from oracle.unet import group_norm, silu as silu_ref
    g = torch.Generator(device="cpu").manual_seed(6)
    c = c0 + c1
    x0 = (torch.randn(b, hw, c0, generator=g) * 2 + 0.5).to(DEV)
    x1 = (torch.randn(b, hw, c1, generator=g) - 1.0).to(DEV) if c1 else None
    sc = (1 + 0.1 * torch.randn(c, generator=g)).to(DEV)
    bi = (0.1 * torch.randn(c, generator=g)).to(DEV)
    s0 = _slab_stats_ref(x0.view(b * hw, c0))
    s1 = _slab_stats_ref(x1.view(b * hw, c1)) if c1 else None
    outs = []
    for mode in ("slabs", "two_pass"):
        ws = torch.full((ops.groupnorm_workspace_floats(b, hw, c),), float("nan"), device=DEV)
        y = torch.zeros(b, hw, c, dtype=torch.bfloat16, device=DEV)
        yf = torch.zeros(b, hw, c, device=DEV)
        raw = torch.zeros(b, hw, c, dtype=torch.bfloat16, device=DEV)
        kw = dict(stats0=s0, stats1=s1) if mode == "slabs" else {}
        ops.groupnorm_fwd(x0, sc, bi, ws, b, hw, c0, x1=x1, c1=c1, silu=silu, y_bf16=y, y_f32=yf, raw_bf16=raw, **kw)
        torch.cuda.synchronize()
        outs.append((y, yf, raw))
    x = x0 if x1 is None else torch.cat([x0, x1], dim=-1)
    ref = group_norm(x.view(b, hw, 1, c), sc, bi).view(b, hw, c)
    if silu:
        ref = silu_ref(ref)
    for y, yf, raw in outs:
        assert (yf - ref).abs().max().item() < 2e-4
        assert rel_err(y, ref) < 4e-3
        assert torch.equal(raw, bf(x))
    assert (outs[0][1] - outs[1][1]).abs().max().item() < 2e-5


@pytest.mark.parametrize("m,c", [(64, 64), (1000, 320), (4096, 1280), (777, 640), (154, 1024), (65536, 320)])
def test_layernorm_fwd(m, c):
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(6)
    x = (torch.randn(m, c, generator=g) * 3 + 1).to(DEV)
    sc = (1 + 0.1 * torch.randn(c, generator=g)).to(DEV)
    bi = (0.1 * torch.randn(c, generator=g)).to(DEV)
    y = torch.zeros(m, c, dtype=torch.bfloat16, device=DEV)
    st = torch.zeros(m, 2, device=DEV)
    ops.layernorm_fwd(x, sc, bi, y, m, c, stats=st)
    ref = torch.nn.functional.layer_norm(x, (c,), sc, bi, 1e-5)
    assert rel_err(y, ref) < 4e-3
    assert (st[:, 0] - x.mean(-1)).abs().max().item() < 1e-5
    assert (st[:, 1] * x.std(-1, unbiased=False) - 1).abs().max().item() < 1e-3


# --------------------------------------------------------------- small layers ----
def test_conv_in_out_dense_upsample():
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(7)
    b, h, c = 3, 16, 64
    lat = torch.randn(b, 4, h, h, generator=g).to(DEV)
    w = torch.randn(3, 3, 4, c, generator=g).to(DEV) / 6
    bias = torch.randn(c, generator=g).to(DEV)
    y = torch.zeros(b * h * h, c, device=DEV)
    st = torch.full(ops.gn_stats_shape(b * h * h, c), float("nan"), device=DEV)
    ops.conv_in(lat, w, bias, y, b, 4, h, h, c, gn_stats=st)
    ref = torch.nn.functional.conv2d(lat, w.permute(3, 2, 0, 1), bias, padding=1).permute(0, 2, 3, 1).reshape(b * h * h, c)
    assert (y - ref).abs().max().item() < 1e-4
    assert (st - _slab_stats_ref(y)).abs().max().item() < 1e-4
    x = torch.randn(b, h, h, c, generator=g).to(DEV)
    w2 = torch.randn(3, 3, c, 4, generator=g).to(DEV) / 24
    b2 = torch.randn(4, generator=g).to(DEV)
    o = torch.zeros(b, 4, h, h, device=DEV)
    ops.conv_out(x, w2, b2, o, b, h, h, c, 4)
    ref2 = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), w2.permute(3, 2, 0, 1), b2, padding=1)
    assert (o - ref2).abs().max().item() < 1e-4
    xin = torch.randn(b, 320, generator=g).to(DEV)
    wd = torch.randn(320, 1280, generator=g).to(DEV) / 18
    bd = torch.randn(1280, generator=g).to(DEV)
    yd = torch.zeros(b, 1280, device=DEV)
    ops.dense_small(xin, wd, bd, yd, b, 320, 1280, silu_in=True, silu_out=True)
    refd = torch.nn.functional.silu(torch.nn.functional.silu(xin) @ wd + bd)
    assert (yd - refd).abs().max().item() < 1e-4
    up = torch.zeros(b, 2 * h, 2 * h, c, dtype=torch.bfloat16, device=DEV)
    ops.upsample2x_bf16(x, up, b, h, h, c)
    assert torch.equal(up, bf(x).repeat_interleave(2, dim=1).repeat_interleave(2, dim=2))
    ts = torch.tensor([981, 1, 500], dtype=torch.int32, device=DEV)
    emb = torch.zeros(b, 320, device=DEV)
    ops.timestep_sincos(ts, emb, b, 320)
    from oracle.unet import timestep_embedding
    refe = timestep_embedding(ts.cpu(), 320, torch.float32)
    assert (emb.cpu() - refe).abs().max().item() < 2e-4


@pytest.mark.parametrize("b,h,c,n", [(2, 16, 64, 64), (3, 32, 128, 160), (5, 8, 128, 256), (1, 64, 320, 320)])
def test_igemm_fat_tile_is_bit_identical(b, h, c, n):
    """Every tile width that divides N must give the same bits (convolution with bias + residual, fp32 and bf16 outputs;
    linear): tile shape is a scheduling choice, never an arithmetic one."""
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(9)
    x = bf(torch.randn(b, h, h, c, generator=g)).to(DEV)
    w = (torch.randn(9 * c, n, generator=g) / math.sqrt(9 * c)).to(DEV)
    bias = torch.randn(n, generator=g).to(DEV)
    res = torch.randn(b * h * h, n, generator=g).to(DEV)
    wt = _prep_w(w)
    outs = []
    for bn in _widths(n):
        o = torch.zeros(b * h * h, n, device=DEV)
        ob = torch.zeros(b * h * h, n, dtype=torch.bfloat16, device=DEV)
        ops.igemm(a0=x, wt=wt, n=n, c0=c, conv=(b, h, h), taps=9, bias=bias, residual=res, out_f32=o, out_bf16=ob, bn=bn)
        outs.append((o, ob))
    torch.cuda.synchronize()
    assert len(outs) >= 2
    for o, ob in outs[1:]:
        assert torch.equal(outs[0][0], o) and torch.equal(outs[0][1], ob)
    ref = _conv_ref(x.float(), bf(w.view(3, 3, c, n)).float(), bias, 1).reshape(b * h * h, n) + res
    assert (outs[1][0] - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())
    # linear
    m, k = b * h * h, c
    a = bf(torch.randn(m, k, generator=g)).to(DEV)
    w2 = (torch.randn(k, n, generator=g) / math.sqrt(k)).to(DEV)
    wt2 = _prep_w(w2)
    lin = []
    for bn in _widths(n):
        o = torch.zeros(m, n, device=DEV)
        ops.igemm(a0=a, wt=wt2, n=n, c0=k, m=m, out_f32=o, bn=bn)
        lin.append(o)
    for o in lin[1:]:
        assert torch.equal(lin[0], o)


@pytest.mark.parametrize("b,h,c0,c1,n,taps,stride", [(2, 16, 64, 0, 64, 9, 1), (3, 32, 128, 64, 160, 9, 1), (5, 8, 128, 0, 256, 9, 1),
                                                     (1, 64, 320, 0, 320, 9, 1), (2, 16, 64, 0, 128, 1, 1), (4, 8, 64, 0, 64, 9, 2)])
def test_igemm_tile_width_is_bit_identical(b, h, c0, c1, n, taps, stride):
    """Two-source / strided / 1x1 convolutions with every epilogue input, and GEGLU: every tile width gives the same bits."""
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(10)
    hi = h * stride
    x0 = bf(torch.randn(b, hi, hi, c0, generator=g)).to(DEV)
    x1 = bf(torch.randn(b, hi, hi, c1, generator=g)).to(DEV) if c1 else None
    cin = c0 + c1
    w = (torch.randn(taps * cin, n, generator=g) / math.sqrt(taps * cin)).to(DEV)
    bias = torch.randn(n, generator=g).to(DEV)
    res = torch.randn(b * h * h, n, generator=g).to(DEV)
    tv = torch.randn(b, n, generator=g).to(DEV)
    wt = _prep_w(w)
    outs = []
    for bn in _widths(n):
        o = torch.zeros(b * h * h, n, device=DEV)
        ob = torch.zeros(b * h * h, n, dtype=torch.bfloat16, device=DEV)
        ops.igemm(a0=x0, a1=x1, wt=wt, n=n, c0=c0, c1=c1, conv=(b, h, h), taps=taps, stride=stride, bias=bias,
                  rowvec=tv, rows_per_sample=h * h, rowvec_ld=n, residual=res, out_f32=o, out_bf16=ob, bn=bn)
        outs.append((o, ob))
    torch.cuda.synchronize()
    assert len(outs) >= 2
    for o, ob in outs[1:]:
        assert torch.equal(outs[0][0], o) and torch.equal(outs[0][1], ob)
    # linear + GEGLU: 256-, 128- and 64-wide tiles (weights and bias permuted for each width)
    m, k = 1000, 128
    a = bf(torch.randn(m, k, generator=g)).to(DEV)
    w2 = (torch.randn(k, 8 * k, generator=g) / math.sqrt(k)).to(DEV)
    b2 = torch.randn(8 * k, generator=g).to(DEV)
    r = []
    for gbn in (256, 128, 64):
        wt2 = torch.empty(8 * k, k, dtype=torch.bfloat16, device=DEV)
        ops.prep_weight(w2, wt2, k, 8 * k, geglu_bn=gbn)
        bp = torch.empty_like(b2)
        ops.permute_geglu_bias(b2, bp, 8 * k, gbn)
        o = torch.zeros(m, 4 * k, dtype=torch.bfloat16, device=DEV)
        ops.igemm(a0=a, wt=wt2, n=8 * k, c0=k, m=m, bias=bp, out_bf16=o, geglu=True, bn=gbn)
        r.append(o)
    torch.cuda.synchronize()
    assert torch.equal(r[0], r[1]) and torch.equal(r[0], r[2])


@pytest.mark.parametrize("m,k,n", [(4096, 320, 320), (1000, 128, 640), (2048 + 37, 64, 96), (8192, 640, 1280)])
@pytest.mark.parametrize("mode", ["res_f32", "bf16", "res_f32_bf16", "f32", "acc_f32", "rowvec_f32"])
def test_igemm_tma_epilogue_is_bit_identical(m, k, n, mode):
    """Every epilogue combination (residual, row vector, accumulate, fp32 / bf16 outputs) gives the same bits with the default
    tile width and with 32-column tiles, including ragged M and outputs narrower than their row pitch."""
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(11)
    a = bf(torch.randn(m, k, generator=g)).to(DEV)
    w = (torch.randn(k, n, generator=g) / math.sqrt(k)).to(DEV)
    wt = _prep_w(w)
    bias = torch.randn(n, generator=g).to(DEV)
    res = torch.randn(m, n, generator=g).to(DEV) if "res" in mode else None
    rows_per = 64
    tv = torch.randn((m + rows_per - 1) // rows_per, n, generator=g).to(DEV) if "rowvec" in mode else None
    init = torch.randn(m, n + 32, generator=g).to(DEV)    # row pitch wider than N: columns n.. must stay untouched
    outs = []
    for bn in (0, 32):
        o = init.clone() if ("f32" in mode) else None
        ob = torch.full((m, n + 32), 7.0, dtype=torch.bfloat16, device=DEV) if "bf16" in mode else None
        ops.igemm(a0=a, wt=wt, n=n, c0=k, m=m, bias=bias, residual=res, ld_res=n if res is not None else 0,
                  rowvec=tv, rows_per_sample=rows_per if tv is not None else 0, rowvec_ld=n if tv is not None else 0,
                  out_f32=o, out_bf16=ob, ld_out=n + 32, accumulate=(mode == "acc_f32"), bn=bn)
        outs.append((o, ob))
    torch.cuda.synchronize()
    for x, y in zip(outs[0], outs[1]):
        if x is not None:
            assert torch.equal(x, y)
    if outs[1][0] is not None:
        assert torch.equal(outs[1][0][:, n:], init[:, n:])
        ref = a.float() @ bf(w).float() + bias
        if res is not None:
            ref = ref + res
        if tv is not None:
            ref = ref + tv.repeat_interleave(rows_per, 0)[:m]
        if mode == "acc_f32":
            ref = ref + init[:, :n]
        assert (outs[1][0][:, :n] - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())
    if outs[1][1] is not None:
        assert (outs[1][1][:, n:].float() == 7.0).all()


@pytest.mark.parametrize("m,k", [(1000, 128), (4096 + 77, 320)])
@pytest.mark.parametrize("with_aux", [False, True])
def test_igemm_geglu_tma_epilogue_is_bit_identical(m, k, with_aux):
    """GEGLU with 256- and 128-column tiles (weights, bias and pre-activations interleaved per tile width): activations
    and pre-activations bit for bit equal; training keeps the pre-activations (aux), sampling does not."""
    from ddpo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(12)
    a = bf(torch.randn(m, k, generator=g)).to(DEV)
    w2 = (torch.randn(k, 8 * k, generator=g) / math.sqrt(k)).to(DEV)
    b2 = torch.randn(8 * k, generator=g).to(DEV)
    r = []
    for gbn in (256, 128):
        wt2 = torch.empty(8 * k, k, dtype=torch.bfloat16, device=DEV)
        ops.prep_weight(w2, wt2, k, 8 * k, geglu_bn=gbn)
        bp = torch.empty_like(b2)
        ops.permute_geglu_bias(b2, bp, 8 * k, gbn)
        o = torch.full((m, 4 * k), 3.0, dtype=torch.bfloat16, device=DEV)
        aux = torch.full((m, 8 * k), 5.0, dtype=torch.bfloat16, device=DEV) if with_aux else None
        ops.igemm(a0=a, wt=wt2, n=8 * k, c0=k, m=m, bias=bp, out_bf16=o, geglu=True, bn=gbn, aux_bf16=aux)
        r.append((o, _geglu_natural(aux, 8 * k, gbn) if with_aux else None))
    torch.cuda.synchronize()
    assert torch.equal(r[0][0], r[1][0])
    if with_aux:
        assert torch.equal(r[0][1], r[1][1])
    lin = a.float() @ bf(w2[:, :4 * k]).float() + b2[:4 * k]
    gate = a.float() @ bf(w2[:, 4 * k:]).float() + b2[4 * k:]
    ref = lin * torch.nn.functional.gelu(gate, approximate="tanh")
    assert (r[1][0].float() - ref).abs().max().item() < 3e-2 * max(1.0, ref.abs().max().item())
