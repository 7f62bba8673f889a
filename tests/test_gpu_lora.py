"""LoRA mode on the H100: the merge kernel (ops.lora_merge) and the adapter-gradient kernel (ops.lora_grad) at every
shape SD2-base and SD1 use, the U-Net backward in LoRA mode against full fine-tuning on the same bf16 operands, and the
train step / sampler on merged adapters (ratio exactly 1 on an unchanged policy, AdamW and Adafactor)."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))

from ddpo_b200 import ops, unet_spec as S  # noqa: E402

pytestmark = pytest.mark.gpu
F32_ULP = 2.0 ** -23
SUM_TOL = 1e-5       # tests/_layer_check.py: reductions, in units of sum |term|


def _adapted_shapes():
    """(family, k, n) of every adapted kernel of SD2-base and SD1, once each"""
    out = set()
    for fam, cfg in (("sd2", S.SD2_BASE), ("sd1", S.SD1)):
        for _, (k, r), kernel in S.lora_manifest(cfg, 4)[::2]:
            out.add((fam, k, S.param_offsets(cfg)[0][kernel][1][1]))
    return sorted(out)


@pytest.mark.parametrize("rank", [4, 8, 16])
@pytest.mark.parametrize("fam,k,n", _adapted_shapes())
def test_merge_kernel(fam, k, n, rank):
    g = torch.Generator().manual_seed(k * 7 + n + rank)
    w = (torch.randn(k, n, generator=g) / np.sqrt(k)).cuda()
    down = (torch.randn(k, rank, generator=g) / rank).cuda()
    w[0, :4] = -0.0                                    # signed zeros, as a pretrained kernel may hold
    up = torch.zeros(rank, n).cuda()
    # U = 0: bit-identical to prep_weight / prep_weight_dgrad, at a row / column offset inside a packed operand
    ref_f, got_f = torch.zeros(3 * n, k, dtype=torch.bfloat16).cuda(), torch.zeros(3 * n, k, dtype=torch.bfloat16).cuda()
    ref_d, got_d = torch.zeros(k, 3 * n, dtype=torch.bfloat16).cuda(), torch.zeros(k, 3 * n, dtype=torch.bfloat16).cuda()
    ops.prep_weight(w, ref_f, k, n, row_offset=n)
    ops.prep_weight_dgrad(w, ref_d, 1, k, n, ld_dst=3 * n, col_offset=n)
    ops.lora_merge(w, down, up, k, n, rank, fwd=got_f, ldk=k, row_offset=n, dgrad=got_d, ld_dst=3 * n, col_offset=n)
    torch.cuda.synchronize()
    assert torch.equal(got_f.view(torch.int16), ref_f.view(torch.int16))
    assert torch.equal(got_d.view(torch.int16), ref_d.view(torch.int16))
    # U != 0: the bf16 rounding of the fp64 merge, except within the fp32 error of a rounding boundary
    up = (torch.randn(rank, n, generator=g) * 0.05).cuda()
    merged = torch.empty(k, n).cuda()
    ops.lora_merge(w, down, up, k, n, rank, fwd=got_f, ldk=k, row_offset=n, dgrad=got_d, ld_dst=3 * n, col_offset=n,
                   merged=merged)
    torch.cuda.synchronize()
    exact = w.double() + down.double() @ up.double()
    mag = w.double().abs() + down.double().abs() @ up.double().abs()
    slack = (rank + 1) * 2.0 ** -24 * mag
    rounded = exact.to(torch.bfloat16)
    lo, hi = (exact - slack).to(torch.bfloat16), (exact + slack).to(torch.bfloat16)
    clear = lo == hi                                   # no rounding boundary within the slack
    for got in (got_f[n:2 * n].t(), got_d[:, n:2 * n]):
        assert torch.equal(got[clear].view(torch.int16), rounded[clear].view(torch.int16))
        # elsewhere: one of the two bf16 values next to the boundary (rounding is monotone)
        assert ((got >= lo) & (got <= hi)).all()
    assert ((merged.double() - exact).abs() <= slack).all()
    assert (got_f[:n] == 0).all() and (got_f[2 * n:] == 0).all() and (got_d[:, :n] == 0).all()


def _grad_cases():
    """(name, G, m, k, n): every adapter-gradient launch of SD2-base and SD1 at 512 px, at train batch 2 with CFG (U-Net
    batch 4) and at the bench's train pass (train batch 2 x 10 timesteps with CFG: U-Net batch 40)"""
    cases = []
    for fam, cfg in (("sd2", S.SD2_BASE), ("sd1", S.SD1)):
        for hw, c in ((4096, 320), (1024, 640), (256, 1280), (64, 1280)):
            for b in (4, 40):
                cases.append((f"{fam}-qkv-c{c}-hw{hw}-b{b}", 3, b * hw, c, c))
                cases.append((f"{fam}-out-c{c}-hw{hw}-b{b}", 1, b * hw, c, c))
        for c in (320, 640, 1280):
            for b in (4, 40):
                cases.append((f"{fam}-ctxkv-c{c}-b{b}", 2, b * 77, cfg.cross_attention_dim, c))
    return sorted(set(cases))


@pytest.mark.parametrize("rank", [4, 8, 16])
@pytest.mark.parametrize("name,G,m,k,n", _grad_cases(), ids=[c[0] for c in _grad_cases()])
def test_grad_kernel(name, G, m, k, n, rank):
    torch.manual_seed(m + k + n + rank)
    dev = "cuda"
    ld = G * n + 64                                     # dy columns inside a wider buffer (as dqkv / dkv slices)
    x = torch.randn(m, k, device=dev).to(torch.bfloat16)
    dy_buf = (torch.randn(m, ld, device=dev) * 0.1).to(torch.bfloat16)
    dys = [dy_buf[:, i * n:] for i in range(G)]
    downs = [torch.randn(k, rank, device=dev) / rank for _ in range(G)]
    ups = [torch.randn(rank, n, device=dev) * 0.05 for _ in range(G)]
    per = k * rank + rank * n
    buf = torch.randn(64 + G * per + 64, device=dev)   # non-zero prior; guard floats on both sides
    prior = buf.clone()
    dd = [buf[64 + i * per:64 + i * per + k * rank].view(k, rank) for i in range(G)]
    du = [buf[64 + i * per + k * rank:64 + (i + 1) * per].view(rank, n) for i in range(G)]
    ops.lora_grad(x, dys, downs, ups, dd, du, m, k, n, rank, lddy=ld)
    first = buf.clone()
    buf.copy_(prior)
    ops.lora_grad(x, dys, downs, ups, dd, du, m, k, n, rank, lddy=ld)
    torch.cuda.synchronize()
    assert torch.equal(buf, first), "two runs differ"
    assert torch.equal(buf[:64], prior[:64]) and torch.equal(buf[-64:], prior[-64:])
    xd, xa = x.double(), x.double().abs()
    for i in range(G):
        dyd = dy_buf[:, i * n:(i + 1) * n].double()
        D, U = downs[i].double(), ups[i].double()
        old_d = prior[64 + i * per:64 + i * per + k * rank].view(k, rank).double()
        old_u = prior[64 + i * per + k * rank:64 + (i + 1) * per].view(rank, n).double()
        ref_d = xd.t() @ (dyd @ U.t())
        ref_u = (xd @ D).t() @ dyd
        terms_d = xa.t() @ (dyd.abs() @ U.abs().t())
        terms_u = (xa @ D.abs()).t() @ dyd.abs()
        for got, ref, old, terms in ((dd[i], ref_d, old_d, terms_d), (du[i], ref_u, old_u, terms_u)):
            err = (got.double() - old - ref).abs()
            bound = SUM_TOL * terms + 2 * F32_ULP * got.double().abs() + 1e-30
            assert (err <= bound).all(), f"adapter {i}: worst {(err / bound).max().item():.3g} of the bound"


# ------------------------------------------------------------------------------------------ U-Net ----
def _sd2_small_batch_net(lora, seed=0):
    from ddpo_b200.unet import UNet
    cfg = S.SD2_BASE
    net = UNet(cfg, S.init_flat_params(cfg, seed), "cuda")
    if lora:
        net.enable_lora(4, seed=1)
    return net


def _randomise_up(net, scale=0.02, seed=2):
    g = torch.Generator().manual_seed(seed)
    for nm, (off, shp) in net.lora_table.items():
        if nm.endswith("lora_up"):
            n = int(np.prod(shp))
            net.lora_params[off:off + n] = (torch.randn(n, generator=g) * scale).cuda()


def test_unet_lora_backward_data_gradients_match_full_mode_and_adapter_gradients_match_the_oracle():
    """SD2-base at 256 px, batch 2: with U != 0, every data gradient of the LoRA-mode backward is bit-identical to full
    fine-tuning's on the same bf16 operands; the adapter gradients against the fp32 oracle's chain-ruled dW on the merged
    weights meet the full-model gradient bounds of test_gpu_sd2_parity.py"""
    from oracle.unet import UNetOracle
    torch.manual_seed(0)
    lat = torch.randn(2, 4, 32, 32)
    ts = torch.tensor([50, 700], dtype=torch.int32)
    ctx = torch.randn(2, 77, 1024)
    probe = torch.randn(2, 4, 32, 32)
    lo = _sd2_small_batch_net(True)
    _randomise_up(lo)
    lo.enable_training()
    lo.refresh_weights()
    fu = _sd2_small_batch_net(False)
    fu.enable_training()
    for key in lo.w:
        fu.w[key].copy_(lo.w[key])
    for key in lo.wd:
        fu.wd[key].copy_(lo.wd[key])
    dbg = []
    for net in (lo, fu):
        net._dbg = {}
        net.prepare_context(ctx.cuda())
        tape = []
        net.forward(lat.cuda(), ts.cuda(), tape=tape)
        net.backward(tape, probe.cuda())
        torch.cuda.synchronize()
        dbg.append(net._dbg)
    assert dbg[0].keys() == dbg[1].keys() and len(dbg[0]) > 20
    for nm in dbg[0]:
        assert torch.equal(dbg[0][nm], dbg[1][nm]), nm
    # oracle: fp32 autograd on the merged weights
    merged = lo.merged_params().cpu()
    kern = {nm[: -len("/lora_down")] + "/kernel" for nm in lo.lora_table if nm.endswith("lora_down")}
    views = {k: (v.clone().requires_grad_() if k in kern else v) for k, v in S.views(merged, S.SD2_BASE).items()}
    out = UNetOracle(S.SD2_BASE, views)(lat, ts.long(), ctx)
    (out * probe).sum().backward()
    got, ref = [], []
    for kn in sorted(kern):
        base = kn[: -len("/kernel")]
        dW = views[kn].grad.double()
        ref += [(dW @ lo.lp(base + "/lora_up").double().cpu().t()).flatten(),
                (lo.lp(base + "/lora_down").double().cpu().t() @ dW).flatten()]
        got += [lo.lg(base + "/lora_down").double().cpu().flatten(), lo.lg(base + "/lora_up").double().cpu().flatten()]
    got, ref = torch.cat(got), torch.cat(ref)
    cos = float(got @ ref / (got.norm() * ref.norm()))
    ratio = float(got.norm() / ref.norm())
    print(f"adapter gradient vs oracle: cosine {cos:.5f}, norm ratio {ratio:.4f}")
    assert cos > 0.995 and abs(ratio - 1) < 5e-2


# ------------------------------------------------------------------------------- sampler + train ----
def _tiny_pipeline(lora_rank):
    from ddpo_b200.diffusers_patch import DDIMScheduler, StableDiffusionPipeline
    from ddpo_b200.unet import UNet
    cfg = S.TINY
    net = UNet(cfg, S.init_flat_params(cfg, 0), "cuda")
    if lora_rank:
        net.enable_lora(lora_rank, seed=4)
    sched = DDIMScheduler(1000, 0.00085, 0.012, "scaled_linear", None, False, 1, "epsilon", device="cuda")
    return net, sched, StableDiffusionPipeline(net, sched, vae_scale_factor=8)


def _sample(pipe, net, sched, seed):
    g = torch.Generator().manual_seed(11)
    emb = torch.randn(2, 77, S.TINY.cross_attention_dim, generator=g).cuda()
    neg = torch.randn(1, 77, S.TINY.cross_attention_dim, generator=g).expand(2, -1, -1).contiguous().cuda()
    state = sched.create_state()
    out = pipe(emb, neg, {"unet": net.params, "scheduler": state}, (0, seed), 3, 128, 128, 5.0, 1.0)
    torch.cuda.synchronize()
    return out, emb, neg, state


@pytest.mark.parametrize("opt", ["adamw", "adafactor"])
def test_sampler_and_train_step_on_merged_adapters(opt):
    from ddpo_b200.training import policy_gradient as pg
    net0, sched0, pipe0 = _tiny_pipeline(0)
    net, sched, pipe = _tiny_pipeline(4)
    (f0, l0, _, lp0, _), *_ = _sample(pipe0, net0, sched0, 7)
    (final, lat, nxt, lps, ts), emb, neg, state = _sample(pipe, net, sched, 7)
    assert torch.equal(final, f0) and torch.equal(lat, l0) and torch.equal(lps, lp0)      # U = 0: same policy
    tx = pg.AdamWConfig(learning_rate=1e-2) if opt == "adamw" else pg.AdafactorConfig(learning_rate=1e-2)
    ts_state = pg.AccumulatingTrainState(apply_fn=net, tx=tx)
    assert net.grads is None and ts_state.params is net.lora_params
    st = sched.set_timesteps(state, 3)

    def step(lat, nxt, lps, ts, emb, neg):
        batch = {"latents": lat[:, 0].contiguous(), "next_latents": nxt[:, 0].contiguous(), "ts": ts[:, 0].contiguous(),
                 "log_probs": lps[:, 0].contiguous(), "advantages": torch.tensor([1.0, -1.0], device="cuda"),
                 "prompt_embeds": emb, "uncond_embeds": neg}
        _, info = pg.train_step(ts_state, batch, st, sched, True, 5.0, 1.0, 1e-4, True)
        torch.cuda.synchronize()
        return info

    p_unet = net.params.clone()
    w_before = {key: t.clone() for key, t in list(net.w.items()) + [("wd:" + k, v) for k, v in net.wd.items()]}
    info = step(lat, nxt, lps, ts, emb, neg)
    assert float(info["approx_kl"]) == 0.0 and float(info["clipfrac"]) == 0.0
    ups = torch.cat([net.lp(nm).flatten() for nm in net.lora_table if nm.endswith("lora_up")])
    assert (ups != 0).any() and torch.equal(net.params, p_unet)                            # adapters moved, U-Net frozen
    # the update re-merged exactly the adapted layers' operands, forward and dgrad layouts
    w_after = dict(list(net.w.items()) + [("wd:" + k, v) for k, v in net.wd.items()])
    adapted = ("/attn1/qkv", "/attn1/to_out_0", "/attn2/q", "/attn2/kv", "/attn2/to_q", "/attn2/to_out_0")
    for key, before in w_before.items():
        assert torch.equal(w_after[key], before) != key.endswith(adapted), key
    # the same seed as before the update: the merged policy samples a different trajectory ...
    (final, lat, nxt, lps, ts), *_ = _sample(pipe, net, sched, 7)
    assert not torch.equal(lps, lp0)
    # ... which trains exactly on-policy
    info = step(lat, nxt, lps, ts, emb, neg)
    assert float(info["approx_kl"]) == 0.0 and float(info["clipfrac"]) == 0.0


# ---------------------------------------------------------------------------------------- epoch ----
def _epoch(lora_rank, savepath):
    """one DDPO epoch of random SD2-base at 512 px through the driver -> (out, models, peak device bytes)"""
    from ddpo_b200 import utils
    from ddpo_b200.pipeline import policy_gradient as PG
    from ddpo_b200.training import policy_gradient as pg
    pg._GRAPHS.clear()
    models = utils.load_unet(None, pretrained_model="random:stabilityai/stable-diffusion-2-base", device="cuda", seed=0)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    argv = ["--dataset", "compressed_animals", "--pretrained_model", "random:stabilityai/stable-diffusion-2-base",
            "--resolution", "512", "--sample_batch_size", "2", "--num_sample_batches_per_epoch", "1",
            "--n_inference_steps", "4", "--train_batch_size", "1", "--train_macro", "2", "--num_train_epochs", "1",
            "--save_freq", "1" if lora_rank else "100", "--learning_rate", "1e-3", "--savepath", savepath, "--seed", "3",
            "--lora_rank", str(lora_rank)]
    out = PG.main(argv, models=models, max_epochs=1, save_last=bool(lora_rank))
    torch.cuda.synchronize()
    return out, models, torch.cuda.max_memory_allocated()


def test_ddpo_epoch_sd2_base_lora_against_full_fine_tuning(tmp_path, monkeypatch):
    """the same DDPO epoch of random SD2-base at 512 px in full mode and with --lora_rank 4: LoRA mode leaves the U-Net
    untouched, allocates no U-Net gradient, saves the merged U-Net, and its peak device memory is lower by at least the
    full mode's gradient buffer plus its AdamW state"""
    from ddpo_b200 import utils
    from ddpo_b200.training import policy_gradient as pg
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv(utils.serialization.ALLOW_RANDOM_ENV, "1")
    out, models, peak_full = _epoch(0, "full")
    st = out["state"]
    state_bytes = st.grad_acc.numel() * 4 + st.opt_state["mu"].numel() * 2 + st.opt_state["nu"].numel() * 4
    assert st.grad_acc is models[0].unet.grads and st.step >= 1
    del out, models, st
    pg._GRAPHS.clear()
    gc.collect()
    torch.cuda.empty_cache()

    out, models, peak_lora = _epoch(4, "lora")
    net, st = models[0].unet, out["state"]
    p0 = S.init_flat_params(S.SD2_BASE, 0)   # the random-init weights load_unet builds at seed 0
    assert torch.equal(models[1]["unet"].cpu(), p0) and torch.equal(net.params.cpu(), p0)    # the U-Net is frozen
    assert net.grads is None and net.lora_rank == 4 and st.params is net.lora_params and st.step >= 1
    assert not torch.equal(st.params.cpu(), S.init_lora_params(S.SD2_BASE, 4, seed=3))      # the adapters trained
    info = out["history"][0]["infos"][0]
    assert info["approx_kl"][0] == 0.0 and np.isfinite(out["history"][0]["mean_reward"])
    tree = utils.restore_checkpoint(os.path.join("logs/compressed-animals/lora", "checkpoints"))
    assert torch.equal(utils.flat_from_tree(tree, S.SD2_BASE), net.merged_params().cpu())    # the merged U-Net
    print(f"one DDPO epoch, random SD2-base at 512 px: peak device memory full {peak_full / 1e9:.2f} GB, LoRA r=4 "
          f"{peak_lora / 1e9:.2f} GB; gradient buffer + AdamW state {state_bytes / 1e9:.2f} GB "
          f"({torch.cuda.get_device_name()})")
    assert peak_full - peak_lora >= state_bytes
