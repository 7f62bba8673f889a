"""LoRA mode on the CPU: the adapter table, the fp64 closed forms the GPU tests of the adapter gradients rely on, and
dry runs of the DDPO epoch driver with ``--lora_rank 4`` on the CPU ops emulator (tests/_lora_emulator.py), on one
rank and on two gloo ranks."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from ddpo_b200 import unet_spec as S  # noqa: E402


# ------------------------------------------------------------------------------------ adapter table ----
@pytest.mark.parametrize("cfg,per_rank", [(S.SD2_BASE, 207488), (S.SD1, 199296)], ids=["sd2", "sd1"])
@pytest.mark.parametrize("rank", [4, 8, 16])
def test_adapter_table(cfg, per_rank, rank):
    table, total = S.lora_offsets(cfg, rank)
    assert total == per_rank * rank == sum(int(np.prod(s)) for _, s in table.values())
    if rank == 4:
        assert total == {S.SD2_BASE: 829952, S.SD1: 797184}[cfg]
    ptable, _ = S.param_offsets(cfg)
    n_blocks = sum(1 for k in ptable if k.endswith("/attn1/to_q/kernel"))
    assert len(table) == n_blocks * 2 * 4 * 2 == 16 * 16
    prev_end = 0
    for name, (off, shape) in table.items():
        assert off % 64 == 0 and off >= prev_end
        prev_end = off + int(np.prod(shape))
        base, leaf = name.rsplit("/", 1)
        k, n = ptable[base + "/kernel"][1]
        assert shape == ((k, rank) if leaf == "lora_down" else (rank, n)), name
        assert base.rsplit("/", 1)[1] in S.LORA_PROJECTIONS and base.split("/")[-2] in ("attn1", "attn2")
    # cross-attention k / v take the text context
    ctx_k = [s for nm, (_, s) in table.items() if "/attn2/to_k/lora_down" in nm]
    assert all(s == (cfg.cross_attention_dim, rank) for s in ctx_k)


@pytest.mark.parametrize("rank", [0, 1, 2, 3, 5, 32, -4])
def test_ranks_outside_4_8_16_are_rejected(rank):
    with pytest.raises(ValueError):
        S.lora_offsets(S.TINY, rank)


def test_adapter_init():
    flat = S.init_lora_params(S.SD2_BASE, 4, seed=5)
    assert torch.equal(flat, S.init_lora_params(S.SD2_BASE, 4, seed=5))
    table, _ = S.lora_offsets(S.SD2_BASE, 4)
    downs = torch.cat([flat[o:o + int(np.prod(s))] for nm, (o, s) in table.items() if nm.endswith("lora_down")])
    ups = torch.cat([flat[o:o + int(np.prod(s))] for nm, (o, s) in table.items() if nm.endswith("lora_up")])
    assert (ups == 0).all() and abs(float(downs.std()) - 0.25) < 2e-3 and abs(float(downs.mean())) < 2e-3


# ----------------------------------------------------------------------------- fp64 closed forms ----
def test_adapter_gradients_are_chain_ruled_kernel_gradients():
    """d/dD = s dW U^T and d/dU = s D^T dW, with dW the oracle's autograd gradient of the merged kernel W + s D U (fp64,
    tiny U-Net, every adapted kernel); and the emulated lora_grad is that closed form for one projection"""
    from oracle.unet import UNetOracle
    cfg, rank, s = S.TINY, 4, 1.0
    flat = S.init_flat_params(cfg, 0).double()
    views = S.views(flat, cfg)
    g = torch.Generator().manual_seed(3)
    table, _ = S.lora_offsets(cfg, rank)
    ad = {nm: (torch.randn(*shp, generator=g, dtype=torch.float64) * 0.1).requires_grad_() for nm, (_, shp) in table.items()}
    merged = {}
    for nm, t in views.items():
        base = nm[: -len("/kernel")]
        if base + "/lora_down" in ad:
            w = t.clone().requires_grad_()
            merged[nm] = w
        else:
            merged[nm] = t
    lat = torch.randn(2, 4, 16, 16, generator=g, dtype=torch.float64)
    ctx = torch.randn(2, cfg.ctx_len, cfg.cross_attention_dim, generator=g, dtype=torch.float64)
    ts = torch.tensor([10, 500])
    probe = torch.randn(2, 4, 16, 16, generator=g, dtype=torch.float64)
    # dW: gradient wrt the merged kernel (a leaf holding the merged value)
    with torch.no_grad():
        for nm, w in merged.items():
            base = nm[: -len("/kernel")]
            if base + "/lora_down" in ad:
                w.copy_(views[nm] + s * ad[base + "/lora_down"] @ ad[base + "/lora_up"])
    out = UNetOracle(cfg, merged, dtype=torch.float64)(lat, ts, ctx)
    (out * probe).sum().backward()
    # adapter gradients by autograd through W + s D U
    p2 = dict(views)
    for nm in views:
        base = nm[: -len("/kernel")]
        if base + "/lora_down" in ad:
            p2[nm] = views[nm] + s * ad[base + "/lora_down"] @ ad[base + "/lora_up"]
    out2 = UNetOracle(cfg, p2, dtype=torch.float64)(lat, ts, ctx)
    assert torch.allclose(out, out2, rtol=0, atol=1e-12)
    (out2 * probe).sum().backward()
    for nm, w in merged.items():
        base = nm[: -len("/kernel")]
        if base + "/lora_down" not in ad:
            continue
        dW, D, U = w.grad, ad[base + "/lora_down"].detach(), ad[base + "/lora_up"].detach()
        torch.testing.assert_close(ad[base + "/lora_down"].grad, s * dW @ U.t(), rtol=1e-10, atol=1e-12)
        torch.testing.assert_close(ad[base + "/lora_up"].grad, s * D.t() @ dW, rtol=1e-10, atol=1e-12)
    # the emulated kernel: x^T (dy U^T) = (x^T dy) U^T and (x D)^T dy = D^T (x^T dy)
    import _lora_emulator as E
    m, k, n = 40, 64, 32
    x = torch.randn(m, k, generator=g).to(torch.bfloat16)
    dy = torch.randn(m, 3 * n, generator=g).to(torch.bfloat16)
    D, U = torch.randn(k, rank, generator=g), torch.randn(rank, n, generator=g)
    dD, dU = torch.zeros(k, rank), torch.zeros(rank, n)
    E.lora_grad(x, [dy[:, n:]], [D], [U], [dD], [dU], m, k, n, rank, lddy=3 * n)
    dW = x.double().t() @ dy[:, n:2 * n].double()
    torch.testing.assert_close(dD.double(), dW @ U.double().t(), rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(dU.double(), D.double().t() @ dW, rtol=1e-5, atol=1e-4)


# ---------------------------------------------------------------------------- driver dry runs ----
@pytest.fixture()
def emulated(monkeypatch, tmp_path):
    import _lora_emulator as E
    from ddpo_b200 import unet as U, vae as V
    from ddpo_b200.diffusers_patch import pipeline_stable_diffusion as P, scheduling_ddim as SD
    from ddpo_b200.pipeline import policy_gradient as DRV
    from ddpo_b200.training import policy_gradient as PG
    for mod in (U, V, P, SD, PG, DRV):
        monkeypatch.setattr(mod, "ops", E)
    monkeypatch.setattr(U, "Arena", E.CpuArena)
    monkeypatch.setattr(V, "Arena", E.CpuArena)
    monkeypatch.setattr(PG, "USE_CUDA_GRAPH", False)
    PG._GRAPHS.clear()
    monkeypatch.chdir(tmp_path)
    orig = P.StableDiffusionPipeline.__init__

    def no_graph_init(self, *a, **k):
        k["use_cuda_graph"] = False
        orig(self, *a, **k)
    monkeypatch.setattr(P.StableDiffusionPipeline, "__init__", no_graph_init)
    from ddpo_b200 import utils
    return lambda seed=0: utils.load_unet(None, pretrained_model="tiny", device="cpu", seed=seed, text_encoder="stub")


DRIVER_ARGV = ["--dataset", "compressed_animals", "--pretrained_model", "tiny", "--resolution", "128",
               "--sample_batch_size", "2", "--num_sample_batches_per_epoch", "1", "--n_inference_steps", "2",
               "--train_batch_size", "2", "--train_macro", "2", "--num_train_epochs", "2", "--save_freq", "1",
               "--learning_rate", "1e-3", "--seed", "3", "--lora_rank", "4"]


def test_lora_epoch_loop_on_the_emulator(emulated):
    from ddpo_b200 import utils
    from ddpo_b200.pipeline import policy_gradient as DRV
    models = emulated(0)
    p0 = models[1]["unet"].clone()
    out = DRV.main(DRIVER_ARGV + ["--savepath", "run0"], models=models, max_epochs=2)
    net, state = models[0].unet, out["state"]
    assert net.lora_rank == 4 and net.grads is None and state.params is net.lora_params
    assert torch.equal(models[1]["unet"], p0) and torch.equal(net.params, p0)          # the U-Net stays frozen
    init = S.init_lora_params(S.TINY, 4, seed=3)
    assert state.step == 2 and not torch.equal(state.params, init)                     # the adapters trained
    info = out["history"][0]["infos"][0]
    assert info["approx_kl"][0] == 0.0 and info["clipfrac"][0] == 0.0                   # unchanged policy: ratio == 1
    assert out["history"][1]["infos"][0]["approx_kl"][0] == 0.0                         # re-sampled: on-policy again
    # the checkpoint is the merged U-Net: W + D U for every adapted kernel, everything else untouched
    tree = utils.restore_checkpoint(os.path.join("logs/compressed-animals/run0", "checkpoints"))
    saved = utils.flat_from_tree(tree, S.TINY)
    ptable, _ = S.param_offsets(S.TINY)
    ltable = net.lora_table
    expect = p0.clone()
    for nm, (off, shp) in ptable.items():
        base = nm[: -len("/kernel")]
        if base + "/lora_down" in ltable:
            expect[off:off + int(np.prod(shp))] = (p0[off:off + int(np.prod(shp))].view(shp)
                                                   + net.lp(base + "/lora_down") @ net.lp(base + "/lora_up")).reshape(-1)
    assert torch.equal(saved, expect) and not torch.equal(saved, p0)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.timeout(600)
def test_two_rank_lora_driver_keeps_adapters_in_sync(tmp_path):
    port = str(_free_port())
    worker = os.path.join(HERE, "_lora_driver_worker.py")
    procs = [subprocess.Popen([sys.executable, worker, str(r), "2", port, str(tmp_path)], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT) for r in range(2)]
    logs = [p.communicate(timeout=560)[0].decode(errors="replace") for p in procs]
    assert all(p.returncode == 0 for p in procs), "\n".join(l[-1500:] for l in logs)
    r = [np.load(tmp_path / f"lora_rank{i}.npz") for i in range(2)]
    assert int(r[0]["step"]) == int(r[1]["step"]) == 2
    np.testing.assert_array_equal(r[0]["adapters"], r[1]["adapters"])                   # replicas in sync, bit for bit
    assert np.abs(r[0]["adapters"] - S.init_lora_params(S.TINY, 4, seed=3).numpy()).max() > 0
    assert not np.array_equal(r[0]["rewards"], r[1]["rewards"])                         # different samples per rank
    np.testing.assert_array_equal(r[0]["checkpoint"], r[0]["merged"])                   # the saved tree is the merged U-Net
    np.testing.assert_array_equal(r[0]["unet"], S.init_flat_params(S.TINY, 0).numpy())  # frozen
