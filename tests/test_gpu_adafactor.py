"""GPU tests of the fused Adafactor update (``csrc/adafactor.cu``): the kernel against a float64 reference built from
the same fp32 operands (every TINY tensor plus the SD2 shapes, and the whole SD2-base buffer), buffer hygiene and
argument checks, ``train_step`` with ``AdafactorConfig`` against the NumPy reference, and one DDPO epoch of
random-init SD2-base at 512 px with ``--optimizer adafactor``.

Bounds.  The reference takes the kernel's own inputs (fp32 params, gradient and prior state, widened to float64) and
runs the chain in float64.  The kernel sums G and u^2 in fp32 over at most ~100 sequential partials, so the state,
the clip denominator and the parameter scale are within 1e-5 relative.  Each element's update is
p - (lr * pscale * u / denom + wd * p): its two terms carry those relative errors plus a few fp32 roundings, and the
result is rounded to fp32 once.  So |dp - dp_ref| <= 1e-4 * (|lr pscale u / denom| + |wd p|) + 1 ulp(p).  This is
the issue's per-element bound with the magnitude of the two terms in place of their sum, which can cancel."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
import _adafactor_ref as A  # noqa: E402

pytestmark = pytest.mark.gpu

SD2_SHAPES = [(320, 1280), (1280, 320), (640, 640), (3, 3, 640, 320), (1, 1, 320, 320), (960, 320), (320,), (1280,)]


def _layout(shapes, align=64):
    tensors, off = [], 0
    for s in shapes:
        tensors.append((off, tuple(s)))
        off += (int(np.prod(s)) + align - 1) // align * align
    return tensors, off


def _ref_tensor(p, g, leaf, beta, kind, lr, wd):
    """float64 torch restatement of tests/_adafactor_ref.py for one tensor (runs on the device)"""
    G = g * g + 1e-30
    nd = p.dim()
    if kind == 0:
        v = beta * leaf["v"] + (1 - beta) * G
        new, u = {"v": v}, g * v.rsqrt()
    else:
        d1, d0 = (nd - 2, nd - 1) if kind == 1 else (nd - 1, nd - 2)
        vr = beta * leaf["v_row"] + (1 - beta) * G.mean(d0)
        vc = beta * leaf["v_col"] + (1 - beta) * G.mean(d1)
        rcm = vr.mean(d1 - 1 if d1 > d0 else d1, keepdim=True)
        new, u = {"v_row": vr, "v_col": vc}, g * (vr / rcm).rsqrt().unsqueeze(d0) * vc.rsqrt().unsqueeze(d1)
    denom = max(1.0, float(u.pow(2).mean().sqrt()))
    pscale = max(float(p.pow(2).mean()), 1e-6) ** 0.5
    step_term, decay = u / denom * lr * pscale, wd * p
    return p - (step_term + decay), new, denom, pscale, step_term.abs() + decay.abs()


def _ulp(x):
    a = x.abs()
    return torch.nextafter(a, torch.full_like(a, float("inf"))) - a


def _update_and_check(tensors, n, plan, p, g, state, step, grad_scale, lr, wd, max_norm=1.0):
    """one kernel update, checked against the float64 reference; returns (clipped, worst error / bound)"""
    from ddpo_b200 import ops
    p0, g0, s0 = p.clone(), g.clone(), state.clone()
    ws = torch.full((plan.workspace_floats,), float("nan"), device="cuda")
    sumsq, norm = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    ops.grad_sumsq(g, ops.optim_workspace(p.device), sumsq)
    ops.clip_adafactor(p, g, state, plan, ws, sumsq, grad_scale, max_norm, lr, wd, step, norm_out=norm)
    torch.cuda.synchronize()
    assert float(g.abs().max()) == 0.0                                     # grad_acc zeroed, padding included
    gh = g0.double() * grad_scale
    gn = float(gh.norm())
    np.testing.assert_allclose(norm.item(), gn, rtol=1e-5)
    clipped = not gn < max_norm
    if clipped:
        gh = gh / gn * max_norm
    beta = 1.0 - step ** -0.8
    before, after = plan.state_views(s0), plan.state_views(state)
    inside = torch.zeros(n, dtype=torch.bool, device="cuda")
    worst = {"state": 0.0, "stats": 0.0, "dp": 0.0}
    stats = ws[:2 * len(tensors)].double().cpu().numpy()
    for t, (off, shape) in enumerate(tensors):
        k = int(np.prod(shape))
        inside[off:off + k] = True
        pt = p0[off:off + k].double().view(shape)
        leaf = {name: v.double() for name, v in before[t].items()}
        pn, new, denom, pscale, mag = _ref_tensor(pt, gh[off:off + k].view(shape), leaf, beta, plan.kinds[t], lr, wd)
        for name, v in new.items():
            worst["state"] = max(worst["state"], float(((after[t][name].double() - v).abs() / v.abs()).max()) / 1e-5)
        worst["stats"] = max(worst["stats"], abs(stats[2 * t] - denom) / denom / 1e-5,
                             abs(stats[2 * t + 1] - pscale) / pscale / 1e-5)
        dp = p[off:off + k].double() - pt.reshape(-1)
        dref = pn.reshape(-1) - pt.reshape(-1)
        bound = 1e-4 * mag.reshape(-1) + _ulp(p0[off:off + k]).double()
        worst["dp"] = max(worst["dp"], float(((dp - dref).abs() / bound).max()))
    assert torch.equal(p[~inside], p0[~inside])                            # padding floats of p untouched
    assert max(worst.values()) <= 1.0, worst
    return clipped, worst


def _buffers(tensors, n, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    p = torch.full((n,), 7.0, device="cuda")                               # padding sentinel
    for i, (off, shape) in enumerate(tensors):
        k = int(np.prod(shape))
        p[off:off + k] = 0.0 if i == len(tensors) - 1 else torch.randn(k, device="cuda", generator=gen) * 0.05
    return p, gen


def _grads(n, scale, gen):
    return torch.randn(n, device="cuda", generator=gen) * (scale / np.sqrt(n))


def _small_case():
    """every TINY tensor, the SD2 shapes, a factored tensor whose gradient stays zero and an all-zero tensor (last)"""
    from ddpo_b200 import unet_spec as S
    return _layout([s for _, s in S.param_manifest(S.TINY)] + SD2_SHAPES + [(256, 512), (256,)])


def test_kernel_matches_fp64_reference_over_steps():
    from ddpo_b200 import ops
    tensors, n = _small_case()
    plan = ops.adafactor_plan(tensors, n)
    p, gen = _buffers(tensors, n, 0)
    state = torch.rand(plan.state_floats, device="cuda", generator=gen) + 0.5     # non-zero prior state
    branches, worst = set(), {}
    for step, sc in ((1, 1e-4), (2, 5.0), (3, 1e-3), (10, 20.0), (1000, 1e-2)):
        g = _grads(n, sc, gen)
        g[~_inside(tensors, n)] = 3.0 if step == 1 else 0.0                   # non-zero gradient padding
        off, shape = tensors[-2]
        g[off:off + int(np.prod(shape))] = 0.0                                # v = 1e-30 exactly at every step
        clipped, w = _update_and_check(tensors, n, plan, p, g, state, step, 0.5, 1e-2, 1e-2)
        branches.add(clipped)
        worst = {k: max(worst.get(k, 0.0), v) for k, v in w.items()}
    assert branches == {True, False}
    print(f"adafactor kernel vs fp64, worst error / bound: {worst}")


def _inside(tensors, n):
    m = torch.zeros(n, dtype=torch.bool, device="cuda")
    for off, shape in tensors:
        m[off:off + int(np.prod(shape))] = True
    return m


def test_fp64_torch_reference_equals_numpy_reference():
    """the device-side float64 reference above is the NumPy restatement tests/_adafactor_ref.py"""
    tensors, n = _layout(SD2_SHAPES)
    rng = np.random.default_rng(0)
    p, g = rng.standard_normal(n) * 0.05, rng.standard_normal(n) * 1e-3
    st = A.AdafactorState(tensors, np.float64)
    want, _, _ = A.clip_adafactor_update(p, g, tensors, st, lr=1e-2, wd=1e-2, max_norm=1e9, dtype=np.float64)
    for off, shape in tensors:
        k = int(np.prod(shape))
        fd = A.factored_dims(shape)
        kind = 0 if fd is None else (1 if fd[1] == len(shape) - 1 else 2)
        leaf = {name: torch.zeros(v.shape, dtype=torch.float64) for name, v in
                A.AdafactorState([(0, shape)], np.float64).leaves[0].items()}
        pn, *_ = _ref_tensor(torch.from_numpy(p[off:off + k].reshape(shape)),
                             torch.from_numpy(g[off:off + k].reshape(shape)), leaf, 0.0, kind, 1e-2, 1e-2)
        np.testing.assert_allclose(pn.numpy().reshape(-1), want[off:off + k], rtol=1e-13, atol=1e-16)


def test_rerun_is_bit_identical_and_bad_buffers_are_refused():
    from ddpo_b200 import _lib, ops
    tensors, n = _small_case()
    plan = ops.adafactor_plan(tensors, n)
    p, gen = _buffers(tensors, n, 1)
    g = _grads(n, 2.0, gen)
    state = torch.rand(plan.state_floats, device="cuda", generator=gen)
    sumsq = torch.zeros(1, device="cuda")
    ops.grad_sumsq(g, ops.optim_workspace(p.device), sumsq)
    outs = []
    for _ in range(2):
        pp, gg, ss = p.clone(), g.clone(), state.clone()
        ws = torch.zeros(plan.workspace_floats, device="cuda")
        ops.clip_adafactor(pp, gg, ss, plan, ws, sumsq, 0.5, 1.0, 1e-2, 1e-4, 7)
        outs.append((pp, gg, ss, ws[:2 * len(tensors)]))
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    ws = torch.zeros(plan.workspace_floats, device="cuda")
    big_p, big_g = torch.zeros(n + 8, device="cuda"), torch.zeros(n + 8, device="cuda")
    big_p[1:n + 1], big_g[1:n + 1] = p, g
    cases = [
        (big_p[1:n + 1], big_g[1:n + 1], state, ws, "aligned"),                 # 4-byte, not 16-byte aligned
        (p.clone(), g.clone(), state[:-1], ws, "state needs"),                  # short state
        (p.clone(), g.clone(), state, ws[:-1], "state needs"),                  # short workspace
        (big_p[:n + 4], big_g[:n + 4], state, ws, "plan is for"),               # buffer of another size
    ]
    for pp, gg, ss, ww, msg in cases:
        before = [t.clone() for t in (pp, gg, ss, ww)]
        with pytest.raises(_lib.DdpoError, match=msg):
            ops.clip_adafactor(pp, gg, ss, plan, ww, sumsq, 0.5, 1.0, 1e-2, 1e-4, 7)
        torch.cuda.synchronize()
        for a, b in zip((pp, gg, ss, ww), before):
            assert torch.equal(a, b)


def test_full_sd2_base_three_updates():
    from ddpo_b200 import ops, unet_spec as S
    table, n = S.param_offsets(S.SD2_BASE)
    tensors = list(table.values())
    assert len(tensors) == 686 and n >= 865_910_724
    plan = ops.adafactor_plan(tensors, n)
    assert plan.state_floats == 1_896_132
    p = S.init_flat_params(S.SD2_BASE, 0).cuda()
    gen = torch.Generator(device="cuda").manual_seed(11)
    state = torch.zeros(plan.state_floats, device="cuda")
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    branches = set()
    for step, sc in ((1, 0.3), (2, 4.0), (3, 0.05)):
        g = _grads(n, sc, gen)
        clipped, worst = _update_and_check(tensors, n, plan, p, g, state, step, 1.0, 1e-3, 1e-4)
        branches.add(clipped)
        print(f"SD2-base update {step}: worst error / bound {worst}")
        del g
    assert branches == {True, False}
    # optimizer memory: the state (7.6 MB) and the workspace, against AdamW's 6 bytes per parameter
    extra = (plan.state_floats + plan.workspace_floats) * 4
    print(f"SD2-base Adafactor state + workspace: {extra / 1e6:.1f} MB (AdamW mu + nu: {6 * n / 1e9:.2f} GB); "
          f"allocated after the updates {(torch.cuda.memory_allocated() - m0) / 1e9:.2f} GB above the start")
    assert extra < 0.02 * 6 * n


def test_train_step_adafactor_update_matches_reference(monkeypatch):
    from ddpo_b200 import ops
    from ddpo_b200.training import policy_gradient as pg
    sys.path.insert(0, os.path.dirname(__file__))
    from test_gpu_training import _batch, _sample
    pg.USE_CUDA_GRAPH = True
    pg._GRAPHS.clear()
    cfg, flat, emb, neg, net, sched, st, out = _sample()
    state = pg.AccumulatingTrainState(apply_fn=net, tx=pg.AdafactorConfig(learning_rate=1e-3, weight_decay=1e-4))
    assert set(state.opt_state) == {"count", "state"} and state.opt_state["state"].numel() == 1_606_468
    seen = []
    orig = ops.clip_adafactor

    def spy(params, grad_acc, st_, plan, ws, sumsq, grad_scale, *a, **k):
        seen.append((params.cpu().numpy().copy(), grad_acc.cpu().numpy() * np.float32(grad_scale)))
        return orig(params, grad_acc, st_, plan, ws, sumsq, grad_scale, *a, **k)
    monkeypatch.setattr(ops, "clip_adafactor", spy)
    pg.train_step(state, _batch(out, emb, neg, 0, [1.0, -1.0]), st, sched, True, 5.0, 1.0, 1e-4, False)
    pg.train_step(state, _batch(out, emb, neg, 2, [0.3, 2.0]), st, sched, True, 5.0, 1.0, 1e-4, False)
    state, info = pg.train_step(state, _batch(out, emb, neg, 1, [-0.5, 0.5]), st, sched, True, 5.0, 1.0, 1e-4, True)
    torch.cuda.synchronize()
    assert len(seen) == 1 and state.step == 1 and state.n_acc == 0 and float(net.grads.abs().max()) == 0.0
    p0, gmean = seen[0]
    tensors = list(net.table.values())
    ref = A.AdafactorState(tensors)
    want, gn, _ = A.clip_adafactor_update(p0, gmean, tensors, ref, lr=1e-3, wd=1e-4, max_norm=1.0)
    np.testing.assert_allclose(state.last_grad_norm.item(), gn, rtol=1e-5)
    got = net.params.cpu().numpy()
    assert np.abs(got - p0).max() > 1e-5
    np.testing.assert_allclose(got, want, rtol=0, atol=3e-7)
    for name, leaf in zip(net.table, ref.leaves):
        for k, v in state.adafactor_leaves()[name].items():
            np.testing.assert_allclose(v.cpu().numpy(), leaf[k], rtol=2e-5)
    state, info = pg.train_step(state, _batch(out, emb, neg, 1, [-0.5, 0.5]), st, sched, True, 5.0, 1.0, 1e-4, False)
    assert info["approx_kl"].item() > 0.0


def _epoch(model, optimizer, savepath):
    from ddpo_b200 import utils
    from ddpo_b200.pipeline import policy_gradient as PG
    from ddpo_b200.training import policy_gradient as pg
    pg._GRAPHS.clear()
    models = utils.load_unet(None, pretrained_model=model, device="cuda", seed=0)
    p0 = models[1]["unet"].clone()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    argv = ["--dataset", "compressed_animals", "--pretrained_model", model, "--resolution", "512",
            "--sample_batch_size", "2", "--num_sample_batches_per_epoch", "1", "--n_inference_steps", "4",
            "--train_batch_size", "1", "--train_macro", "2", "--num_train_epochs", "1", "--save_freq", "100",
            "--learning_rate", "1e-5", "--savepath", savepath, "--seed", "3", "--optimizer", optimizer]
    out = PG.main(argv, models=models, max_epochs=1, save_last=False)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    moved = not torch.equal(models[1]["unet"], p0)
    info = out["history"][0]["infos"][0]
    res = (out["state"], info, moved, peak, out["history"][0]["mean_reward"])
    del models, out
    pg._GRAPHS.clear()
    return res


def test_ddpo_epoch_sd2_base_adafactor(tmp_path, monkeypatch):
    from ddpo_b200 import utils
    from ddpo_b200.training import policy_gradient as pg
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv(utils.serialization.ALLOW_RANDOM_ENV, "1")
    model = "random:stabilityai/stable-diffusion-2-base"
    state, info, moved, peak_af, reward = _epoch(model, "adafactor", "af")
    assert isinstance(state.tx, pg.AdafactorConfig) and "mu" not in state.opt_state and state.step >= 1
    assert info["approx_kl"][0] == 0.0 and moved and np.isfinite(reward)
    del state
    torch.cuda.empty_cache()
    _, _, _, peak_adamw, _ = _epoch(model, "adamw", "aw")
    line = (f"one DDPO epoch, random SD2-base at 512 px: peak device memory adafactor {peak_af / 1e9:.2f} GB, "
            f"adamw {peak_adamw / 1e9:.2f} GB ({torch.cuda.get_device_name()})")
    print(line)
    assert peak_af < peak_adamw
