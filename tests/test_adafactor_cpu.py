"""CPU tests of optimizer=adafactor: the NumPy restatement (tests/_adafactor_ref.py) against the third-party pin
``transformers.optimization.Adafactor`` and against closed forms where optax and transformers differ, the host planner
of ``csrc/adafactor.cu`` on every model config, the CPU emulation of the update, and the DDPO epoch driver with
``--optimizer adafactor`` on one and on two gloo ranks."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(__file__))
import _adafactor_ref as A  # noqa: E402

PIN_SHAPES = [(320, 1280), (1280, 320), (640, 640), (3, 3, 640, 320), (1, 1, 320, 320), (320,), (128,)]


def _layout(shapes, align=64):
    tensors, off = [], 0
    for s in shapes:
        tensors.append((off, tuple(s)))
        off += (int(np.prod(s)) + align - 1) // align * align
    return tensors, off


def test_reference_matches_transformers_adafactor_float64():
    """steps 2-6 of the chain against transformers' Adafactor (wd = 0, where both compute the same update); the
    global-norm clip is applied to the pin's input with optax's formula, once below and once above max_norm"""
    from transformers.optimization import Adafactor
    rng = np.random.default_rng(0)
    tensors, n = _layout(PIN_SHAPES)
    p0 = rng.standard_normal(n) * 0.05
    p0[tensors[-1][0]:tensors[-1][0] + 128] = 0.0                   # all-zero tensor: the 1e-3 parameter-scale floor
    lr, max_norm = 1e-2, 1.0
    st = A.AdafactorState(tensors, np.float64)
    p_ref = p0.copy()
    tp = [torch.tensor(p0[o:o + int(np.prod(s))].reshape(s), dtype=torch.float64, requires_grad=True) for o, s in tensors]
    opt = Adafactor(tp, lr=lr, scale_parameter=True, relative_step=False, warmup_init=False, beta1=None,
                    clip_threshold=1.0, decay_rate=-0.8, eps=(1e-30, 1e-3), weight_decay=0.0)
    scales = [1e-3, 10.0, 1e-4, 3.0, 1e-3, 50.0]
    block_clipped = clipped = unclipped = False
    for step, sc in enumerate(scales):
        g = rng.standard_normal(n) * sc / np.sqrt(n)
        g[tensors[0][0] + 7] *= 300.0 if step == 1 else 1.0          # a spike: rms(u) > 1 in the factored tensor
        gn = np.sqrt(np.sum(g ** 2))
        clipped |= gn >= max_norm
        unclipped |= gn < max_norm
        gc = g if gn < max_norm else g / gn * max_norm
        prev = p_ref.copy()
        p_ref, _, stats = A.clip_adafactor_update(p_ref, g, tensors, st, lr=lr, wd=0.0, max_norm=max_norm,
                                                  dtype=np.float64)
        block_clipped |= any(d > 1.0 for d, _ in stats)
        if step == 0:
            assert stats[-1][1] == 1e-3
        for t, (o, s) in zip(tp, tensors):
            t.grad = torch.tensor(gc[o:o + int(np.prod(s))].reshape(s), dtype=torch.float64)
        opt.step()
        for t, (o, s) in zip(tp, tensors):
            k = int(np.prod(s))
            d_ref = p_ref[o:o + k] - prev[o:o + k]
            d_pin = t.detach().numpy().reshape(-1) - prev[o:o + k]
            ulp = np.spacing(np.abs(prev[o:o + k])) + np.spacing(np.abs(p_ref[o:o + k]))   # the subtraction's rounding
            assert (np.abs(d_ref - d_pin) <= 1e-10 * np.abs(d_ref).max() + ulp).all(), (step, s)
    assert clipped and unclipped and block_clipped


def test_shapes_optax_leaves_unfactored():
    """optax factors only when the second-largest dim is >= 128: conv_in / conv_out and [64, 128] keep a full v, and
    the first update (beta = 0, v = g^2 + 1e-30) is then -lr * pscale * sign(g) (transformers would factor them)"""
    for s in [(3, 3, 4, 320), (3, 3, 320, 4), (64, 128), (127, 4096)]:
        assert A.factored_dims(s) is None, s
    assert A.factored_dims((128, 128)) == (0, 1) and A.factored_dims((3, 3, 640, 320)) == (3, 2)
    tensors, n = _layout([(64, 128), (3, 3, 4, 320)])
    rng = np.random.default_rng(1)
    p, g = rng.standard_normal(n) * 0.1, rng.standard_normal(n) * 1e-3
    st = A.AdafactorState(tensors, np.float64)
    new, _, stats = A.clip_adafactor_update(p, g, tensors, st, lr=1e-3, wd=0.0, dtype=np.float64)
    for (o, s), (denom, pscale) in zip(tensors, stats):
        k = int(np.prod(s))
        assert denom == 1.0 and st.leaves[0]["v"].shape == (64, 128)
        np.testing.assert_allclose(new[o:o + k] - p[o:o + k], -1e-3 * pscale * np.sign(g[o:o + k]), rtol=1e-12)
        np.testing.assert_allclose(pscale, np.sqrt(np.mean(p[o:o + k] ** 2)), rtol=1e-15)


def test_weight_decay_is_not_scaled_by_the_learning_rate():
    tensors, n = _layout([(320, 1280), (320,)])
    rng = np.random.default_rng(2)
    p, g = rng.standard_normal(n), rng.standard_normal(n)
    st = A.AdafactorState(tensors, np.float64)
    new, _, _ = A.clip_adafactor_update(p, g, tensors, st, lr=0.0, wd=1e-4, dtype=np.float64)
    for o, s in tensors:
        k = int(np.prod(s))
        np.testing.assert_allclose(new[o:o + k], p[o:o + k] * (1 - 1e-4), rtol=1e-15)


def test_first_step_uses_beta_zero_and_later_steps_decay():
    assert A.beta_t(0) == 0.0
    np.testing.assert_allclose(A.beta_t(1), 1 - 2 ** -0.8, rtol=1e-7)
    tensors, n = _layout([(256, 512), (40,)])
    rng = np.random.default_rng(3)
    g = rng.standard_normal(n)
    st = A.AdafactorState(tensors, np.float64)
    st.leaves[0]["v_row"][:] = 5.0                 # prior state: ignored when beta = 0
    st.leaves[1]["v"][:] = 5.0
    A.clip_adafactor_update(np.ones(n), g * 1e-3, tensors, st, lr=1e-3, wd=0.0, dtype=np.float64)
    G = (g * 1e-3) ** 2 + 1e-30
    o, s = tensors[0]
    np.testing.assert_allclose(st.leaves[0]["v_row"], G[o:o + 256 * 512].reshape(s).mean(axis=1), rtol=1e-14)
    o, s = tensors[1]
    np.testing.assert_allclose(st.leaves[1]["v"], G[o:o + 40], rtol=1e-15)


def test_row_col_mean_is_per_tap():
    """rank-1 G per tap with tap scales 1e4 apart: the factored estimate is exact per tap, so the first update is
    -lr * pscale * sign(g) everywhere; an rcm over the whole tensor would scale taps by up to 1e2"""
    s = (3, 3, 256, 128)
    rng = np.random.default_rng(4)
    a = 10.0 ** rng.uniform(-2, 2, (3, 3, 1, 1))
    x, y = rng.uniform(0.5, 2, (1, 1, 256, 1)), rng.uniform(0.5, 2, (1, 1, 1, 128))
    g = (np.sqrt(a * x * y) * rng.choice([-1.0, 1.0], s) * 1e-4).reshape(-1)
    tensors, n = _layout([s])
    p = rng.standard_normal(n)
    st = A.AdafactorState(tensors, np.float64)
    k = int(np.prod(s))
    assert n == k
    new, _, stats = A.clip_adafactor_update(p, g, tensors, st, lr=1e-3, wd=0.0, dtype=np.float64)
    np.testing.assert_allclose(new[:k] - p[:k], -1e-3 * stats[0][1] * np.sign(g[:k]), rtol=1e-9)


# ------------------------------------------------------------------ the host planner ----
EXPECTED_STATE = {"SD2_BASE": 1896132, "SD1": 1887940, "TINY": 1606468}


@pytest.mark.parametrize("name", ["SD2_BASE", "SD1", "TINY", "SMALL"])
def test_planner_factoring_state_and_tiles(name):
    from ddpo_b200 import ops, unet_spec as S
    cfg = getattr(S, name)
    table, n = S.param_offsets(cfg)
    tensors = list(table.values())
    plan = ops.adafactor_plan(tensors, n)
    st = A.AdafactorState(tensors)
    for t, (off, shape) in enumerate(tensors):
        fd = A.factored_dims(shape)
        want = 0 if fd is None else (1 if fd == (len(shape) - 2, len(shape) - 1) else 2)
        assert fd is None or set(fd) == {len(shape) - 2, len(shape) - 1}
        assert plan.kinds[t] == want, (t, shape, fd)
        assert plan.state_shapes(t) == {k: v.shape for k, v in st.leaves[t].items()}
    assert plan.state_floats == sum(v.size for leaf in st.leaves for v in leaf.values())
    if name in EXPECTED_STATE:
        assert plan.state_floats == EXPECTED_STATE[name]
    # state offsets: leaf by leaf, in tensor order, without gaps
    flat = [o for offs in plan.state_offsets for o in offs if o >= 0]
    sizes = [v.size for leaf in st.leaves for v in leaf.values()]
    assert flat == list(np.cumsum([0] + sizes[:-1]))
    # every tensor element lies in exactly one tile: per tensor-tap the tiles form a grid over [0, R) x [0, C)
    T, L = plan.tensors, plan.tiles
    covered = 0
    for t, (off, shape) in enumerate(tensors):
        rows = L[L[:, 0] == t]
        taps, R, C = int(T[t, 3]), int(T[t, 4]), int(T[t, 5])
        assert int(T[t, 0]) == off and taps * R * C == int(np.prod(shape))
        for k in range(taps):
            tk = rows[rows[:, 1] == k]
            r_iv = sorted({(int(a), int(b)) for a, b in tk[:, 2:4]})
            c_iv = sorted({(int(a), int(b)) for a, b in tk[:, 4:6]})
            assert len(tk) == len(r_iv) * len(c_iv)
            for iv, ext in ((r_iv, R), (c_iv, C)):
                assert iv[0][0] == 0 and all(iv[i][0] + iv[i][1] == iv[i + 1][0] for i in range(len(iv) - 1))
                assert iv[-1][0] + iv[-1][1] == ext
            assert len({(int(a), int(b)) for a, b in tk[:, [2, 4]]}) == len(tk)
            covered += int((tk[:, 3] * tk[:, 5]).sum())
    assert covered == sum(int(np.prod(s)) for _, s in tensors)
    # the padding is in no tile; the grad_acc zero ranges cover exactly the padding
    pad = [(int(a), int(b)) for a, b in L[:, 6:8] if b > a]
    spans = sorted(pad + [(o, o + int(np.prod(s))) for o, s in tensors])
    assert spans[0][0] == 0 and spans[-1][1] == n and all(spans[i][1] == spans[i + 1][0] for i in range(len(spans) - 1))
    if name in ("TINY", "SMALL"):   # brute force: count every element's tiles
        cnt = np.zeros(n, np.int32)
        for row in L:
            t = int(row[0])
            if t < 0:
                continue
            off, C = int(T[t, 0]), int(T[t, 5])
            base = off + int(row[1]) * int(T[t, 4]) * C
            idx = base + (int(row[2]) + np.arange(int(row[3])))[:, None] * C + int(row[4]) + np.arange(int(row[5]))
            cnt[idx.reshape(-1)] += 1
        inside = np.zeros(n, bool)
        for o, s in tensors:
            inside[o:o + int(np.prod(s))] = True
        assert (cnt[inside] == 1).all() and (cnt[~inside] == 0).all()


def test_planner_refuses_bad_layouts_and_writes_nothing():
    from ddpo_b200 import _lib, ops
    with pytest.raises(_lib.DdpoError, match="two largest dims"):
        ops.adafactor_plan([(0, (320, 3, 320))], 307200)
    with pytest.raises(_lib.DdpoError, match="two largest dims"):
        ops.adafactor_plan([(0, (512, 3, 3, 256))], 512 * 9 * 256)
    with pytest.raises(_lib.DdpoError, match="aligned"):
        ops.adafactor_plan([(0, (130, 130))], 130 * 132)
    with pytest.raises(_lib.DdpoError, match="overlaps"):
        ops.adafactor_plan([(0, (256,)), (128, (256,))], 1024)
    with pytest.raises(_lib.DdpoError, match="larger than the buffer"):
        ops.adafactor_plan([(0, (256, 256))], 1024)
    ops.adafactor_plan([(0, (320, 3, 100))], 96000)          # second-largest 100 < 128: unfactored, accepted
    sizes = np.full(3, -7, np.int64)
    offs, nd, dims = np.zeros(1, np.int64), np.array([3], np.int32), np.array([320, 3, 320], np.int64)
    plan = np.full(64, -7, np.int64)
    st = _lib.lib().ddpo_adafactor_plan(1, offs.ctypes.data, nd.ctypes.data, dims.ctypes.data, 307200, 128,
                                        plan.ctypes.data, 64, sizes.ctypes.data, None)
    assert st != 0 and (sizes == -7).all() and (plan == -7).all()


# ------------------------------------------------------------------ emulator and drivers ----
def test_emulator_update_matches_reference():
    import _adafactor_emulator as E
    from ddpo_b200 import unet_spec as S
    table, n = S.param_offsets(S.TINY)
    tensors = list(table.values())
    plan = E.adafactor_plan(tensors, n)
    p = S.init_flat_params(S.TINY, 0)
    state = torch.zeros(plan.state_floats)
    ws = torch.zeros(plan.workspace_floats)
    ref = A.AccumulatingTrainState(p.numpy(), tensors, lr=1e-3, wd=1e-4, max_norm=1.0)
    rng = np.random.default_rng(5)
    for step, sc in enumerate([1e-6, 1.0, 1e-5], 1):
        g = (rng.standard_normal(n) * sc).astype(np.float32)
        acc = torch.from_numpy(g.copy())
        sumsq = (acc.double() ** 2).sum().float().reshape(1)
        E.clip_adafactor(p, acc, state, plan, ws, sumsq, 1.0, 1.0, 1e-3, 1e-4, step)
        ref.apply_gradients(g, True)
        assert (acc == 0).all()
        np.testing.assert_allclose(p.numpy() - ref.params, 0, atol=2e-6 * 1e-3)
        for views, leaf in zip(plan.state_views(state), ref.opt.leaves):
            for k in leaf:
                np.testing.assert_allclose(views[k].numpy(), leaf[k], rtol=1e-5)


@pytest.fixture()
def emulated(monkeypatch, tmp_path):
    import _cpu_ops_emulator as E
    from ddpo_b200 import unet as U, vae as V
    from ddpo_b200.diffusers_patch import pipeline_stable_diffusion as P, scheduling_ddim as SD
    from ddpo_b200.pipeline import policy_gradient as DRV
    from ddpo_b200.training import policy_gradient as PG
    import _adafactor_emulator as AE
    monkeypatch.setattr(E, "adafactor_plan", AE.adafactor_plan, raising=False)
    monkeypatch.setattr(E, "clip_adafactor", AE.clip_adafactor, raising=False)
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
    return E


def test_ddpo_epoch_driver_with_adafactor_matches_reference(emulated, monkeypatch):
    """the driver builds AdafactorConfig from the command line; every update it issues equals the reference chain fed
    the same accumulated gradient, and the state it ends with is the reference's after all its updates"""
    from ddpo_b200 import unet_spec, utils
    from ddpo_b200.pipeline import policy_gradient as DRV
    from ddpo_b200.training import policy_gradient as PG
    E = emulated
    models = utils.load_unet(None, pretrained_model="tiny", device="cpu", seed=0, text_encoder="stub")
    table, n = unet_spec.param_offsets(unet_spec.TINY)
    tensors = list(table.values())
    ref = A.AdafactorState(tensors)
    seen = []
    orig = E.clip_adafactor

    def checked(params, grad_acc, state, plan, ws, sumsq, grad_scale, max_norm, lr, wd, step, norm_out=None):
        p0, g0 = params.numpy().copy(), grad_acc.numpy() * np.float32(grad_scale)
        orig(params, grad_acc, state, plan, ws, sumsq, grad_scale, max_norm, lr, wd, step, norm_out)
        want, _, _ = A.clip_adafactor_update(p0, g0, tensors, ref, lr=2e-4, wd=1e-4, max_norm=1.0)
        seen.append(step)
        np.testing.assert_allclose(params.numpy() - want, 0, atol=1e-9)
        for views, leaf in zip(plan.state_views(state), ref.leaves):
            for k in leaf:
                np.testing.assert_allclose(views[k].numpy(), leaf[k], rtol=1e-5)
    monkeypatch.setattr(E, "clip_adafactor", checked)
    argv = ["--dataset", "compressed_animals", "--pretrained_model", "tiny", "--resolution", "128",
            "--sample_batch_size", "2", "--num_sample_batches_per_epoch", "2", "--n_inference_steps", "2",
            "--train_batch_size", "2", "--train_macro", "2", "--num_train_epochs", "2", "--save_freq", "100",
            "--learning_rate", "2e-4", "--savepath", "run_af", "--seed", "3", "--optimizer", "adafactor"]
    out = DRV.main(argv, models=models, max_epochs=2, save_last=False)
    state = out["state"]
    assert isinstance(state.tx, PG.AdafactorConfig) and seen == [1, 2, 3, 4] and state.step == 4
    assert set(state.opt_state) == {"count", "state"} and state.opt_state["state"].numel() == 1606468
    leaves = state.adafactor_leaves()
    assert set(leaves["conv_in/kernel"]) == {"v"} and leaves["up_blocks_0/resnets_0/time_emb_proj/kernel"]["v_row"].shape == (128,)
    info = out["history"][0]["infos"][0]
    assert info["approx_kl"][0] == 0.0 and info["approx_kl"][1] > 0.0


def test_unknown_optimizer_names_both_choices(emulated):
    from ddpo_b200 import utils
    from ddpo_b200.pipeline import policy_gradient as DRV
    models = utils.load_unet(None, pretrained_model="tiny", device="cpu", seed=0, text_encoder="stub")
    with pytest.raises(ValueError, match="adamw, adafactor"):
        DRV.main(["--pretrained_model", "tiny", "--optimizer", "sgd", "--savepath", "x"], models=models, max_epochs=1)


@pytest.mark.timeout(600)
def test_two_rank_driver_with_adafactor_keeps_replicas_identical(tmp_path):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = str(s.getsockname()[1])
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_adafactor_driver_worker.py")
    procs = [subprocess.Popen([sys.executable, worker, str(r), "2", port, str(tmp_path)], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT) for r in range(2)]
    logs = [p.communicate(timeout=560)[0].decode(errors="replace") for p in procs]
    assert all(p.returncode == 0 for p in procs), "\n".join(l[-1500:] for l in logs)
    r = [np.load(tmp_path / f"af_rank{i}.npz") for i in range(2)]
    assert int(r[0]["step"]) == int(r[1]["step"]) == 2
    np.testing.assert_array_equal(r[0]["params"], r[1]["params"])
    np.testing.assert_array_equal(r[0]["state"], r[1]["state"])
    assert not np.array_equal(r[0]["rewards"], r[1]["rewards"])
    from ddpo_b200 import unet_spec
    assert np.abs(r[0]["params"] - unet_spec.init_flat_params(unet_spec.TINY, 0).numpy()).max() > 1e-6
