"""SD1.x on the GPU: attention forward and backward at head dims 40, 80 and 160 (64 as the control) with the pitches
unet.py uses, the rejection of unsupported head dims and layouts, a small SD1-shaped U-Net against the oracle, the full
SD1 U-Net (859,520,964 parameters) against the fp32 oracle, and one epoch of the DDPO driver on a random-init SD1.

The whole-model numbers are printed, stored as test properties (``pytest --junitxml=...`` writes them out) and, when
``$DDPO_SD1_PARITY_LOG`` names a file, appended to it.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _layer_check import (ATT_L2, ATT_MAX, BF16, F32, F32_L2, F32_MAX, Guarded, _current_node, _record, check_close,  # noqa: E402,F401
                          check_sum, rnd)
from ddpo_b200.unet_spec import UNetConfig  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
G, ETA, T = 5.0, 1.0, 50
DIMS = (40, 64, 80, 160)
# (head_dim, n, heads): every SD1 token count (64 x 64 latents: 4096 .. 64; TINY-sized 16, 4; a ragged 300) at 8 heads,
# and an odd head count
CASES = [(d, n, 8) for d in DIMS for n in (4096, 1024, 256, 64, 16, 4, 300)] + [(d, n, 3) for d in DIMS for n in (300, 16)]
L = 77


def _id(c):
    return "d{}-n{}-h{}".format(*c)


def _heads(t, rows, heads, d):
    """[b * n, >= heads * d] -> [b, heads, n, d] float64"""
    return t[:, :heads * d].double().reshape(-1, rows, heads, d).permute(0, 2, 1, 3)


def _flat(t):
    b, h, n, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(b * n, h * d)


def _reference(q, k, v, do, n, nk, heads, d):
    """float64 O, LSE and (dQ, dK, dV) of softmax(Q K^T / sqrt(d)) V from the bf16 operands the kernel reads"""
    qq, kk, vv = (_heads(t, r, heads, d).requires_grad_(True) for t, r in ((q, n), (k, nk), (v, nk)))
    s = qq @ kk.transpose(-1, -2) * d ** -0.5
    o = torch.softmax(s, -1) @ vv
    lse = torch.logsumexp(s, -1)
    grads = None
    if do is not None:
        o.backward(_heads(do, n, heads, d))
        grads = [_flat(t.grad) for t in (qq, kk, vv)]
    return _flat(o.detach()), lse.detach(), grads


def _operands(kind, b, n, heads, d, seed):
    """self: q/k/v column slices of one [b n, 3C] qkv buffer; cross: q [b n, C], k/v slices of [b 77, 2C]"""
    c = heads * d
    g = torch.Generator().manual_seed(seed)
    if kind == "self":
        qkv = rnd(g, b * n, 3 * c).to(BF16).to(DEV)
        return dict(q=qkv, k=qkv[:, c:], v=qkv[:, 2 * c:], ldq=3 * c, ldk=3 * c, ldv=3 * c, nk=n, g=g)
    q = rnd(g, b * n, c).to(BF16).to(DEV)
    kv = rnd(g, b * L, 2 * c).to(BF16).to(DEV)
    return dict(q=q, k=kv, v=kv[:, c:], ldq=c, ldk=2 * c, ldv=2 * c, nk=L, g=g)


def _fwd(op, b, n, heads, d, s0=0, extra_cols=64):
    """forward into guarded out / lse for samples [s0, s0 + b)"""
    from ddpo_b200 import ops
    c, nk = heads * d, op["nk"]
    qr, kr = slice(s0 * n, (s0 + b) * n), slice(s0 * nk, (s0 + b) * nk)
    out = Guarded(b * n, c, BF16, DEV, extra_cols=extra_cols)
    lse = Guarded(b * heads, n, F32, DEV)
    ops.attention_fwd(op["q"][qr], op["k"][kr], op["v"][kr], out.arg, b, heads, n, nk, op["ldq"], op["ldk"], op["ldv"],
                      out.ld, lse=lse.view, head_dim=d)
    torch.cuda.synchronize()
    out.check("out")
    lse.check("lse")
    return out.view.clone(), lse.view.clone()


@pytest.mark.parametrize("kind", ["self", "cross"])
@pytest.mark.parametrize("d,n,heads", CASES, ids=[_id(c) for c in CASES])
def test_attention_fwd_head_dims(kind, d, n, heads):
    b = 2
    op = _operands(kind, b, n, heads, d, seed=d * 7 + n + heads)
    out, lse = _fwd(op, b, n, heads, d)
    ref, ref_lse, _ = _reference(op["q"], op["k"], op["v"], None, n, op["nk"], heads, d)
    check_close("out", out, ref, ATT_MAX, ATT_L2)
    check_close("lse", lse, ref_lse.reshape(b * heads, n), F32_MAX, F32_L2)
    # the last sample alone gives the same bits as inside the batch; a rerun too
    out1, lse1 = _fwd(op, 1, n, heads, d, s0=b - 1)
    assert torch.equal(out1, out[(b - 1) * n:]) and torch.equal(lse1, lse[(b - 1) * heads:])
    assert all(torch.equal(x, y) for x, y in zip(_fwd(op, b, n, heads, d), (out, lse)))


def _bwd(op, out, do, lse, b, n, heads, d, s0=0):
    from ddpo_b200 import ops
    c, nk = heads * d, op["nk"]
    qr, kr = slice(s0 * n, (s0 + b) * n), slice(s0 * nk, (s0 + b) * nk)
    delta = Guarded(b * heads, n, F32, DEV)
    if op["ldq"] == 3 * c:   # self: one [b n, 3C] gradient buffer (pitch widened by a sentinel block)
        dqkv = Guarded(b * n, 3 * c, BF16, DEV, extra_cols=64)
        buf = dqkv.buf
        dq, dk, dv, lddq = buf, buf[:, c:], buf[:, 2 * c:], dqkv.ld
        lddk = lddv = lddq
        guards = [dqkv]
    else:                    # cross: dq [b n, C], dk / dv slices of one [b 77, 2C]
        gq, gkv = Guarded(b * n, c, BF16, DEV), Guarded(b * nk, 2 * c, BF16, DEV)
        dq, dk, dv, lddq, lddk, lddv = gq.view, gkv.view, gkv.view[:, c:], c, 2 * c, 2 * c
        guards = [gq, gkv]
    ops.attention_bwd(op["q"][qr], op["k"][kr], op["v"][kr], out[qr], do[qr], lse[s0 * heads:(s0 + b) * heads], delta.view,
                      dq, dk, dv, b, heads, n, nk, op["ldq"], op["ldk"], op["ldv"], c, c, lddq, lddk, lddv, head_dim=d)
    torch.cuda.synchronize()
    for gd in guards + [delta]:
        gd.check("attention_bwd")
    if len(guards) == 1:
        v = guards[0].view
        grads = [v[:, :c].clone(), v[:, c:2 * c].clone(), v[:, 2 * c:].clone()]
    else:
        grads = [guards[0].view.clone(), guards[1].view[:, :c].clone(), guards[1].view[:, c:].clone()]
    return grads, delta.view.clone()


@pytest.mark.parametrize("kind", ["self", "cross"])
@pytest.mark.parametrize("d,n,heads", CASES, ids=[_id(c) for c in CASES])
def test_attention_bwd_head_dims(kind, d, n, heads):
    b = 2
    c = heads * d
    op = _operands(kind, b, n, heads, d, seed=d * 11 + n + heads)
    out, lse = _fwd(op, b, n, heads, d, extra_cols=0)
    do = rnd(op["g"], b * n, c).to(BF16).to(DEV)
    grads, delta = _bwd(op, out, do, lse, b, n, heads, d)
    _, _, ref = _reference(op["q"], op["k"], op["v"], do, n, op["nk"], heads, d)
    for name, got, r in zip(("dq", "dk", "dv"), grads, ref):
        check_close(name, got, r, ATT_MAX, ATT_L2)
    prod = (out.double() * do.double()).reshape(b, n, heads, d)
    check_sum("delta", delta.reshape(b, heads, n).permute(0, 2, 1), prod.sum(-1), prod.abs().sum(-1))
    # deterministic: a rerun gives the same bits, and so does the last sample alone
    grads2, delta2 = _bwd(op, out, do, lse, b, n, heads, d)
    assert all(torch.equal(x, y) for x, y in zip(grads + [delta], grads2 + [delta2]))
    alone, delta1 = _bwd(op, out, do, lse, 1, n, heads, d, s0=b - 1)
    nk = op["nk"]
    assert torch.equal(alone[0], grads[0][(b - 1) * n:])
    assert torch.equal(alone[1], grads[1][(b - 1) * nk:]) and torch.equal(alone[2], grads[2][(b - 1) * nk:])
    assert torch.equal(delta1, delta[(b - 1) * heads:])


@pytest.mark.parametrize("d", [48, 96, 0, 256, 32, -64])
def test_attention_rejects_unsupported_head_dims(d):
    from ddpo_b200 import ops
    from ddpo_b200._lib import DdpoError
    b, n, heads = 1, 64, 2
    c = heads * 64
    x = torch.randn(b * n, 3 * c).to(BF16).to(DEV)
    out = Guarded(b * n, c, BF16, DEV)
    lse = Guarded(b * heads, n, F32, DEV)
    with pytest.raises(DdpoError, match="head_dim"):
        ops.attention_fwd(x, x[:, c:], x[:, 2 * c:], out.view, b, heads, n, n, 3 * c, 3 * c, 3 * c, c, lse=lse.view,
                          head_dim=d)
    dg = Guarded(b * n, 3 * c, BF16, DEV)
    delta = Guarded(b * heads, n, F32, DEV)
    with pytest.raises(DdpoError, match="head_dim"):
        ops.attention_bwd(x, x[:, c:], x[:, 2 * c:], x, x, lse.view, delta.view, dg.view, dg.view[:, c:], dg.view[:, 2 * c:],
                          b, heads, n, n, 3 * c, 3 * c, 3 * c, 3 * c, 3 * c, 3 * c, 3 * c, 3 * c, head_dim=d)
    torch.cuda.synchronize()
    for t in (out, lse, dg, delta):
        t.check("rejected call")
        assert torch.equal(t.buf, t.snapshot)


@pytest.mark.parametrize("d", DIMS)
@pytest.mark.parametrize("bad", ["ldq", "ldo", "q_base", "out_base", "lddq", "dk_base", "ld_short"])
def test_attention_rejects_misaligned_layouts(d, bad):
    """a base pointer off 16 bytes or a row pitch that is not a multiple of 8 elements is refused; nothing is written"""
    from ddpo_b200 import ops
    from ddpo_b200._lib import DdpoError
    b, n, heads = 1, 64, 2
    c = heads * d
    ld = 3 * c + 8
    x = torch.randn(b * n + 1, ld + 8).to(BF16).to(DEV)
    out = Guarded(b * n, c + 8, BF16, DEV)
    lse = Guarded(b * heads, n, F32, DEV)
    q = x.reshape(-1)[1:1 + b * n * ld].view(b * n, ld) if bad == "q_base" else x[:b * n, :ld]
    ldq = ld - 4 if bad == "ldq" else (c - 8 if bad == "ld_short" else ld)
    ldo = c + 4 if bad == "ldo" else c + 8
    o = out.buf.reshape(-1)[1:] if bad == "out_base" else out.buf
    fwd_bad = bad in ("ldq", "ldo", "q_base", "out_base", "ld_short")
    if fwd_bad:
        with pytest.raises(DdpoError, match="aligned"):
            ops.attention_fwd(q, q[:, c:], q[:, 2 * c:], o, b, heads, n, n, ldq, ld, ld, ldo, lse=lse.view, head_dim=d)
    else:
        dg = Guarded(b * n, 3 * c + 16, BF16, DEV)
        delta = Guarded(b * heads, n, F32, DEV)
        lddq = 3 * c + 12 if bad == "lddq" else 3 * c + 16
        dk = dg.buf.reshape(-1)[c + 1:] if bad == "dk_base" else dg.buf[:, c:]
        with pytest.raises(DdpoError, match="aligned"):
            ops.attention_bwd(q, q[:, c:], q[:, 2 * c:], out.buf, out.buf, lse.view, delta.view, dg.buf, dk, dg.buf[:, 2 * c:],
                              b, heads, n, n, ld, ld, ld, c + 8, c + 8, lddq, 3 * c + 16, 3 * c + 16, head_dim=d)
        torch.cuda.synchronize()
        for t in (dg, delta):
            assert torch.equal(t.buf, t.snapshot)
    torch.cuda.synchronize()
    for t in (out, lse):
        assert torch.equal(t.buf, t.snapshot)


# ------------------------------------------------------------------ small SD1-shaped U-Net --------------------
SD1_SMALL = UNetConfig(block_out_channels=(320, 320, 320, 320), attention_head_dim=(8, 4, 2, 2), cross_attention_dim=768,
                       use_linear_projection=False, sample_size=16)


def test_sd1_small_unet_forward_matches_oracle_and_is_batch_invariant():
    from ddpo_b200 import unet_spec
    from ddpo_b200.unet import UNet
    from oracle.unet import UNetOracle
    cfg = SD1_SMALL
    flat = unet_spec.init_flat_params(cfg, 0)
    g = torch.Generator().manual_seed(1)
    s = cfg.sample_size
    lat = torch.randn(5, 4, s, s, generator=g)
    ctx = torch.randn(5, cfg.ctx_len, cfg.cross_attention_dim, generator=g)
    ts = torch.tensor([981, 21, 441, 1, 700], dtype=torch.int32)
    net = UNet(cfg, flat, DEV)
    net.prepare_context(ctx[:2].to(DEV))
    eps = net.forward(lat[:2].to(DEV), ts[:2].to(DEV)).clone()
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = UNetOracle(cfg, unet_spec.views(flat, cfg))(lat[:2], ts[:2].long(), ctx[:2])
    rel = ((eps.cpu() - ref).norm() / ref.norm()).item()
    assert rel < 2e-2, rel
    net.prepare_context(ctx.to(DEV))
    eps5 = net.forward(lat.to(DEV), ts.to(DEV))
    torch.cuda.synchronize()
    assert torch.equal(eps5[:2], eps)


def test_sd1_small_unet_backward_matches_oracle():
    from ddpo_b200 import unet_spec
    from ddpo_b200.unet import UNet
    from oracle.unet import UNetOracle
    cfg, batch = SD1_SMALL, 2
    flat = unet_spec.init_flat_params(cfg, 0)
    g = torch.Generator().manual_seed(11)
    s = cfg.sample_size
    lat = torch.randn(batch, 4, s, s, generator=g)
    ctx = torch.randn(batch, cfg.ctx_len, cfg.cross_attention_dim, generator=g)
    ts = torch.tensor([981, 441], dtype=torch.int32)
    d_eps = torch.randn(batch, 4, s, s, generator=g) / (4 * s * s)
    net = UNet(cfg, flat, DEV)
    net.enable_training()
    net.prepare_context(ctx.to(DEV))
    tape = []
    net.forward(lat.to(DEV), ts.to(DEV), tape=tape)
    net.backward(tape, d_eps.to(DEV))
    torch.cuda.synchronize()
    fp = flat.clone().requires_grad_(True)
    UNetOracle(cfg, unet_spec.views(fp, cfg))(lat, ts.long(), ctx).backward(d_eps)
    table, _ = unet_spec.param_offsets(cfg)
    gg, ref = net.grads.cpu(), fp.grad
    tot = ((gg - ref).norm() / ref.norm()).item()
    worst, worst_name = 0.0, None
    for name, (off, shape) in table.items():
        n = int(np.prod(shape))
        a, r = gg[off:off + n], ref[off:off + n]
        if r.norm() > 1e-3 * ref.norm() / np.sqrt(len(table)):
            e = ((a - r).norm() / r.norm()).item()
            if e > worst:
                worst, worst_name = e, name
    assert tot < 4e-2, f"total gradient relative error {tot}"
    assert worst < 0.2, f"worst tensor {worst_name}: {worst}"


# ------------------------------------------------------------------ full SD1 ----------------------------------
def _log(line):
    _record("sd1_parity", line=line)
    path = os.environ.get("DDPO_SD1_PARITY_LOG")
    if path:
        os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
        with open(path, "a") as f:
            f.write(line + "\n")
    print(line)


def _rel(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


@pytest.fixture(scope="module")
def sd1():
    """SD1 on both sides from the same seeded CPU weights; the oracle's first denoising step is computed once."""
    from ddpo_b200 import unet_spec
    from ddpo_b200.diffusers_patch import DDIMScheduler
    from ddpo_b200.unet import UNet
    from oracle import ppo as OPPO, scheduler as OS, threefry
    from oracle.unet import UNetOracle
    import psutil
    torch.set_num_threads(max(1, min(psutil.cpu_count(logical=False) or 8, len(os.sched_getaffinity(0)))))
    cfg = unet_spec.SD1
    flat = unet_spec.init_flat_params(cfg, 0)
    assert sum(int(np.prod(shape)) for _, shape in unet_spec.param_offsets(cfg)[0].values()) == 859_520_964
    onet = UNetOracle(cfg, unet_spec.views(flat, cfg))
    g = torch.Generator().manual_seed(1)
    ctx = torch.randn(2, 77, 768, generator=g)                                   # [uncond ; cond]
    x = threefry.normal(np.array((0, 7), np.uint32), (1, 4, 64, 64)).astype(np.float32)
    key = (0, 11)
    ost = OS.set_timesteps(OS.SD_CONFIG, OS.create_state(OS.SD_CONFIG), T)
    t0 = int(ost.timesteps[0])
    xt = torch.from_numpy(x)
    with torch.no_grad():
        e = onet(torch.cat([xt, xt]), torch.full((2,), t0), ctx).numpy()
    eps = OPPO.cfg_combine(e[:1], e[1:], G)
    prev, _, lp = OS.step(OS.SD_CONFIG, ost, eps, t0, x, key=np.array(key, np.uint32), eta=ETA)
    net = UNet(cfg, flat, DEV)
    sched = DDIMScheduler(1000, 0.00085, 0.012, "scaled_linear", None, False, 1, "epsilon", device=DEV)
    st = sched.set_timesteps(sched.create_state(), T)
    return dict(cfg=cfg, flat=flat, ctx=ctx, x=x, key=key, ost=ost, t0=t0, e=e, prev=prev, lp=np.asarray(lp), net=net,
                sched=sched, st=st)


def test_sd1_denoising_step_matches_oracle(sd1):
    from ddpo_b200 import ops
    s = sd1
    net, st = s["net"], s["st"]
    xg = torch.from_numpy(s["x"]).to(DEV).view(1, -1)
    tdev = torch.tensor([s["t0"]], dtype=torch.int32, device=DEV)
    net.prepare_context(s["ctx"].to(DEV))
    eps_g = net.forward(torch.cat([xg, xg]).view(2, 4, 64, 64), tdev).view(2, -1)
    prev_g, lp_g, lp_s = torch.empty_like(xg), torch.empty(1, device=DEV), torch.empty(1, device=DEV)
    ws = ops.ddim_workspace(1, DEV)
    ac, fa = st.common.alphas_cumprod, st.final_alpha_cumprod
    ops.ddim_step_sample(eps_g[:1], eps_g[1:], xg, ac, tdev, fa, 20, G, ETA, ops.key_tensor([s["key"]], DEV), prev_g, lp_g, ws)
    ops.ddim_logprob_fwd(eps_g[:1], eps_g[1:], xg, torch.from_numpy(s["prev"]).to(DEV).view(1, -1), ac, tdev, fa, 20, G, ETA,
                         lp_s, ws)
    torch.cuda.synchronize()
    eps_rel = _rel(eps_g.cpu().numpy(), s["e"])
    lat_rel = _rel(prev_g.cpu().numpy(), s["prev"])
    lp_o = float(s["lp"].ravel()[0])
    lp_rel = abs(lp_g.item() / lp_o - 1)
    lps_rel = abs(lp_s.item() / lp_o - 1)
    ratio = math.exp(lp_s.item() - lp_o)
    _log(f"SD1 denoise step t={s['t0']}: eps rel-L2 {eps_rel:.3e}  first-step latents rel-L2 "
         f"{lat_rel:.3e}  log_prob (sample mode) rel {lp_rel:.3e}  log_prob of the oracle's x_prev under GPU eps rel "
         f"{lps_rel:.3e}  importance ratio {ratio:.6f}  (log_prob oracle {lp_o:.6f})")
    assert np.isfinite(eps_g.cpu().numpy()).all()
    assert eps_rel < 2.5e-2, f"eps relative L2 error {eps_rel}"
    assert lat_rel < 2.5e-2, f"first-step latents relative L2 error {lat_rel}"
    assert lp_rel < 1e-3, f"per-step log_prob relative error {lp_rel}"
    assert lps_rel < 2e-2 and abs(ratio - 1) < 2e-2, (lps_rel, ratio)


def test_sd1_batch_invariance_of_eps(sd1):
    s = sd1
    net = s["net"]
    xg = torch.from_numpy(s["x"]).to(DEV).view(1, 4, 64, 64)
    tdev = torch.tensor([s["t0"]], dtype=torch.int32, device=DEV)
    net.prepare_context(s["ctx"].to(DEV))
    e2 = net.forward(torch.cat([xg, xg]), tdev).clone()
    g = torch.Generator().manual_seed(9)
    other = torch.randn(2, 4, 64, 64, generator=g).to(DEV)
    octx = torch.randn(2, 77, 768, generator=g).to(DEV)
    ctx6 = torch.cat([s["ctx"][:1].to(DEV), octx, s["ctx"][1:].to(DEV), octx])      # [u(x), u(o0), u(o1), c(x), c(o0), c(o1)]
    net.prepare_context(ctx6)
    e6 = net.forward(torch.cat([xg, other, xg, other]), tdev)
    torch.cuda.synchronize()
    assert torch.equal(e6[0], e2[0]) and torch.equal(e6[3], e2[1])


@pytest.mark.timeout(600)
def test_sd1_ppo_train_step_matches_oracle(sd1):
    from ddpo_b200 import unet_spec
    from ddpo_b200.training import policy_gradient as pg
    from oracle import pipeline as OP, scheduler as OS
    from oracle.unet import UNetOracle
    s = sd1
    cfg = s["cfg"]
    clip = 1e9
    batch_np = {"latents": s["x"], "next_latents": s["prev"], "ts": np.array([s["t0"]], np.int32),
                "log_probs": s["lp"].reshape(1).astype(np.float32), "advantages": np.array([1.0], np.float32),
                "prompt_embeds": s["ctx"][1:].numpy(), "uncond_embeds": s["ctx"][:1].numpy()}
    params = {k: v.clone().requires_grad_(True) for k, v in unet_spec.views(s["flat"], cfg).items()}
    loss, info, lp = OP.train_loss(UNetOracle(cfg, params), OS.SD_CONFIG, s["ost"], batch_np, True, G, ETA, clip)
    loss.backward()
    ref = {k: p.grad for k, p in params.items()}
    pg.USE_CUDA_GRAPH = False
    pg._GRAPHS.clear()
    net = s["net"]
    state = pg.AccumulatingTrainState(apply_fn=net)
    net.grads.zero_()
    batch = {k: torch.as_tensor(v).to(DEV) for k, v in batch_np.items()}
    state, ginfo = pg.train_step(state, batch, s["st"], s["sched"], True, G, ETA, clip, False)
    torch.cuda.synchronize()
    gg = net.grads.cpu()
    table, _ = unet_spec.param_offsets(cfg)
    tot_num = tot_den = dot = na = 0.0
    blocks = {}
    for name, (off, shape) in table.items():
        n = int(np.prod(shape))
        a, r = gg[off:off + n].double(), ref[name].reshape(-1).double()
        d2, r2 = float(((a - r) ** 2).sum()), float((r ** 2).sum())
        tot_num, tot_den = tot_num + d2, tot_den + r2
        dot, na = dot + float((a * r).sum()), na + float((a ** 2).sum())
        b = blocks.setdefault(name.split("/")[0], [0.0, 0.0])
        b[0] += d2
        b[1] += r2
    grad_rel = math.sqrt(tot_num / tot_den)
    cos = dot / math.sqrt(na * tot_den)
    norm_ratio = math.sqrt(na / tot_den)
    _log(f"SD1 PPO train step: loss gpu {ginfo['loss'].item():.6f} oracle {float(loss):.6f}  grad rel-L2 {grad_rel:.3e}  "
         f"cosine {cos:.6f}  |g_gpu|/|g_oracle| {norm_ratio:.4f}")
    for blk, (d2, r2) in blocks.items():
        _log(f"    block {blk:24s} grad rel-L2 {math.sqrt(d2 / r2):.3e}   |g| {math.sqrt(r2):.3e}")
    net.grads.zero_()
    pg.USE_CUDA_GRAPH = True
    assert abs(ginfo["loss"].item() - float(loss)) < 2e-2 * max(1.0, abs(float(loss)))
    assert cos > 0.995 and abs(norm_ratio - 1) < 5e-2, (cos, norm_ratio)
    assert grad_rel < 0.1, grad_rel
    for blk, (d2, r2) in blocks.items():
        assert math.sqrt(d2 / r2) < 0.2, (blk, math.sqrt(d2 / r2))


# ------------------------------------------------------------------ the DDPO driver on SD1 --------------------
def test_ddpo_driver_epoch_on_random_init_sd1(tmp_path, monkeypatch):
    from ddpo_b200 import utils
    from ddpo_b200.pipeline import policy_gradient as PG
    from ddpo_b200.training import policy_gradient as pg
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv(utils.serialization.ALLOW_RANDOM_ENV, "1")
    pg._GRAPHS.clear()
    model = "random:duongna/stable-diffusion-v1-4-flax"
    models = utils.load_unet(None, pretrained_model=model, device="cuda", seed=0)
    p0 = models[1]["unet"].clone()
    argv = ["--dataset", "compressed_animals", "--pretrained_model", model, "--resolution", "512",
            "--sample_batch_size", "2", "--num_sample_batches_per_epoch", "1", "--n_inference_steps", "4",
            "--train_batch_size", "1", "--train_macro", "2", "--num_train_epochs", "1", "--save_freq", "100",
            "--learning_rate", "1e-5", "--savepath", "sd1", "--seed", "3"]
    out = PG.main(argv, models=models, max_epochs=1, save_last=False)
    info = out["history"][0]["infos"][0]
    # 2 samples / train batch 1 = 2 minibatches x (4 timesteps / macro 2) = 4 passes
    assert info["approx_kl"].shape == (4,)
    assert info["approx_kl"][0] == 0.0 and info["approx_kl"][1] == 0.0
    assert info["clipfrac"][0] == 0.0 and info["clipfrac"][1] == 0.0
    assert np.isfinite(out["history"][0]["mean_reward"])
    assert not torch.equal(models[1]["unet"], p0)
