"""CPU tests of the image-symmetry and consistency rewards: the host bicubic coefficient tables against Pillow, the
device preprocessing restated on the CPU against ``clip_vision.preprocess``, the consistency oracle against the
installed ``transformers`` ``CLIPModel``, the host assembly of every new reward on the CPU ops emulator against the
reference restatement (tests/_rewards_ref.py), and the DDPO epoch driver with ``--filter_field mirror`` / ``rotational``."""
import functools
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image, ImageOps

sys.path.insert(0, os.path.dirname(__file__))
import _image_rewards_emulator as IE  # noqa: E402
import _rewards_ref as R  # noqa: E402

from ddpo_b200 import clip_vision as CV, text_encoder as TE  # noqa: E402
from ddpo_b200.training import callbacks as C  # noqa: E402
from oracle import clip_vision as OCV, text_encoder as OTE  # noqa: E402

SIZES = [(512, 224), (512, 128), (512, 64), (512, 32), (128, 224), (64, 224), (32, 224), (256, 224), (768, 224),
         (224, 224)]
TRANSFORMS = {CV.IDENTITY: lambda p: p, CV.MIRROR: ImageOps.mirror, CV.ROT90: lambda p: p.rotate(90),
              CV.ROT180: lambda p: p.rotate(180), CV.ROT270: lambda p: p.rotate(270)}
TINY_TEXT = TE.CLIPTextConfig(vocab_size=49408, hidden_size=128, intermediate_size=256, num_hidden_layers=2,
                              num_attention_heads=2, hidden_act="quick_gelu")


def test_image(kind, s, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (s, s, 3), dtype=np.uint8)
    if kind == "flat":
        return np.full((s, s, 3), 77, np.uint8)
    if kind == "saturated":
        return np.where(rng.random((s, s, 3)) < 0.5, 0, 255).astype(np.uint8)
    a = np.zeros((s, s, 3), np.uint8)              # edges: a bright square and a one-pixel line
    a[s // 4:s // 2, s // 3:2 * s // 3] = 255
    a[:, s - 1 - s // 5] = (255, 0, 128)
    return a


test_image.__test__ = False


def _np_resize(a, w, h, transform):
    x = IE.transformed(a[None], transform)
    if x.shape[2] != w or x.shape[1] == h:
        x = IE.resample_axis(x, 2, CV.resample_table(x.shape[2], w))
    if x.shape[1] != h:
        x = IE.resample_axis(x, 1, CV.resample_table(x.shape[1], h))
    return x[0]


@pytest.mark.parametrize("src,dst", SIZES)
def test_coefficient_tables_equal_pillow_bicubic(src, dst):
    for kind in ("random", "flat", "saturated", "edge"):
        a = test_image(kind, src)
        for t, f in TRANSFORMS.items():
            want = np.array(f(Image.fromarray(a)).resize((dst, dst), Image.BICUBIC))
            np.testing.assert_array_equal(_np_resize(a, dst, dst, t), want, err_msg=f"{kind} transform {t}")


def test_rotation_before_resample_is_not_resample_before_rotation():
    a = test_image("random", 512)
    rot_first = _np_resize(a, 224, 224, CV.ROT90)
    rot_last = np.rot90(_np_resize(a, 224, 224, CV.IDENTITY), 1)
    assert not np.array_equal(rot_first, rot_last)


def test_tables_are_normalised_fixed_point():
    for src, dst in SIZES:
        t = CV.resample_table(src, dst)
        assert t.dtype == np.int32 and t.shape[0] == dst
        assert (t[:, 0] >= 0).all() and (t[:, 0] + t[:, 1] <= src).all()
        assert np.abs(t[:, 2:].sum(1) - (1 << 22)).max() <= t.shape[1]     # rounding of each weight only


@pytest.fixture()
def emu(monkeypatch):
    import _cpu_ops_emulator as E
    IE.install(E)
    for mod in (CV, TE, C):
        monkeypatch.setattr(mod, "ops", E)
    monkeypatch.setattr(CV, "Arena", E.CpuArena)
    monkeypatch.setattr(TE, "Arena", E.CpuArena)
    return E


@pytest.mark.parametrize("shape,size", [((3, 64, 64, 3), 32), ((2, 80, 80, 3), 56), ((2, 56, 56, 3), 56),
                                        ((2, 60, 90, 3), 32), ((2, 512, 512, 3), 224)])
def test_device_preprocess_restatement_is_bit_identical_to_preprocess(emu, shape, size):
    imgs = np.random.default_rng(1).integers(0, 256, shape, dtype=np.uint8)
    got = CV.preprocess_device(torch.from_numpy(imgs), size).numpy()
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got, CV.preprocess(imgs, size))
    if shape[1] == shape[2]:
        for t, f in TRANSFORMS.items():
            want = CV.preprocess(np.stack([np.array(f(Image.fromarray(a))) for a in imgs]), size)
            np.testing.assert_array_equal(CV.preprocess_device(torch.from_numpy(imgs), size, t).numpy(), want)


def test_rotate_90_of_a_non_square_image_is_refused(emu):
    with pytest.raises(ValueError):
        CV.resize_u8(torch.zeros(1, 60, 90, 3, dtype=torch.uint8), 32, 32, CV.ROT90)


def _batch(n=4, s=64, seed=0):
    imgs = np.random.default_rng(seed).random((n, s, s, 3)).astype(np.float32)
    imgs[1] = (imgs[1] + imgs[1][:, ::-1]) / 2                  # mirror-symmetric
    imgs[2] = (imgs[2] + np.rot90(imgs[2], 2)) / 2              # symmetric under rotate(180)
    return imgs


def test_pixel_rewards_equal_the_reference_on_the_emulator(emu):
    imgs = _batch()
    u8 = (imgs * 255).astype(np.uint8)
    for name, ref in (("mirror", R.mirror), ("rotational_corr", R.rotational_corr)):
        fn = C.callback_fns[name](device="cpu")
        s, info = fn(imgs, ["p"] * 4, {})
        want = ref(imgs)
        assert s.dtype == np.float64 and s.shape == (4,) and info == {}
        assert (s == want).all(), (name, s, want)
        assert (fn(u8, ["p"] * 4, {})[0] == s).all()
    fn = C.callback_fns["mirror_corr"](device="cpu")
    s, _ = fn(imgs, ["p"] * 4, {})
    assert s.dtype == np.float32 and s.shape == (4,)
    np.testing.assert_allclose(s, R.mirror_corr(imgs, np.float64), rtol=0, atol=1e-6)
    np.testing.assert_allclose(s, R.mirror_corr(imgs), rtol=0, atol=1e-5)       # the reference's own float32 cov
    assert (fn(u8, ["p"] * 4, {})[0] == s).all()


def test_mirror_wraps_like_numpy_uint8():
    a = np.zeros((1, 2, 2, 3), np.uint8)
    a[0, :, 0] = 3
    a[0, :, 1] = 200                                        # (3 - 200) % 256 = 59, 59^2 % 256 = 153
    assert R.mirror(a)[0] == -153.0


def test_mirror_corr_of_a_flat_image_is_nan(emu):
    imgs = np.zeros((2, 32, 32, 3), np.uint8)
    imgs[1] = test_image("random", 32)
    s, _ = C.callback_fns["mirror_corr"](device="cpu")(imgs, ["p"] * 2, {})
    with np.errstate(invalid="ignore", divide="ignore"):
        want = R.mirror_corr(imgs)
    assert np.isnan(s[0]) and np.isnan(want[0]) and np.isfinite(s[1])


def _emulated_features(tower):
    return lambda px: tower.image_features(torch.from_numpy(np.ascontiguousarray(px))).numpy()


@pytest.mark.parametrize("name,ref", [("rotational", R.rotational), ("thumbnail", R.thumbnail)])
def test_angle_rewards_host_assembly_on_the_emulator(emu, name, ref):
    cfg = CV.VIT_TINY
    fn = C.callback_fns[name](device="cpu", cfg=cfg)
    imgs = _batch(3, 64)
    s, info = fn(imgs, ["p"] * 3, {})
    assert s.dtype == np.float32 and s.shape == (3,) and info == {}
    tower = CV.CLIPImageTower(cfg, device="cpu", seed=0)
    np.testing.assert_allclose(s, ref(imgs, _emulated_features(tower), cfg.image_size), rtol=0, atol=1e-4)
    # and against the fp32 oracle tower (the emulated tower runs bf16 GEMM operands)
    oracle = lambda px: OCV.image_features(CV.views(CV.init_flat_params(cfg, 0, head=False), cfg, head=False), cfg,
                                           torch.from_numpy(np.ascontiguousarray(px))).numpy()
    np.testing.assert_allclose(s, ref(imgs, oracle, cfg.image_size), rtol=0, atol=2.0)
    assert (fn((imgs * 255).astype(np.uint8), ["p"] * 3, {})[0] == s).all()


def test_tower_without_head_has_the_aesthetic_towers_weights():
    cfg = CV.VIT_TINY
    a, b = CV.init_flat_params(cfg, 3), CV.init_flat_params(cfg, 3, head=False)
    va, vb = CV.views(a, cfg), CV.views(b, cfg, head=False)
    assert set(vb) == {k for k in va if not k.startswith("aesthetic/")}
    assert all(torch.equal(va[k], vb[k]) for k in vb)


# ------------------------------------------------------------------ consistency ----
def _oracle_consistency(model, pixels, prompts):
    """fp32 restatement: oracle towers, argmax pooling, bias-free projections, the reference's logits diagonal"""
    ids, pos = model.token_ids(prompts)
    vcfg, tcfg = model.vision.cfg, model.text.cfg
    img = OCV.image_features(CV.views(model.vision.params.cpu(), vcfg, head=False), vcfg, torch.from_numpy(pixels))
    hidden = OTE.encode(TE.views(model.text.params.cpu(), tcfg), tcfg, ids)
    txt = hidden[torch.arange(len(ids)), torch.from_numpy(pos)] @ model.text_projection.cpu()
    return R.consistency(img.double().numpy(), txt.double().numpy(), np.float32(model.logit_scale))


def _hf_clip_model(model):
    tr = pytest.importorskip("transformers")
    vcfg, tcfg = model.vision.cfg, model.text.cfg
    cfg = tr.CLIPConfig(
        text_config=dict(vocab_size=tcfg.vocab_size, hidden_size=tcfg.hidden_size, intermediate_size=tcfg.intermediate_size,
                         num_hidden_layers=tcfg.num_hidden_layers, num_attention_heads=tcfg.num_attention_heads,
                         max_position_embeddings=tcfg.max_position_embeddings, hidden_act=tcfg.hidden_act,
                         layer_norm_eps=tcfg.layer_norm_eps, attention_dropout=0.0, eos_token_id=49407),
        vision_config=dict(hidden_size=vcfg.hidden_size, intermediate_size=vcfg.intermediate_size,
                           num_hidden_layers=vcfg.num_hidden_layers, num_attention_heads=vcfg.num_attention_heads,
                           image_size=vcfg.image_size, patch_size=vcfg.patch_size, hidden_act=vcfg.hidden_act,
                           layer_norm_eps=vcfg.layer_norm_eps, attention_dropout=0.0),
        projection_dim=vcfg.projection_dim, logit_scale_init_value=CV.CLIPConsistency.LOGIT_SCALE_INIT)
    hf = tr.CLIPModel(cfg).eval()
    sd = hf.state_dict()
    pv, pt = CV.views(model.vision.params.cpu(), vcfg, head=False), TE.views(model.text.params.cpu(), tcfg)

    def layers(prefix, fx, p, n):
        for i in range(n):
            b, hb = f"{fx}/encoder/layers/{i}", f"{prefix}.encoder.layers.{i}"
            for ln in ("layer_norm1", "layer_norm2"):
                sd[f"{hb}.{ln}.weight"].copy_(p[f"{b}/{ln}/scale"])
                sd[f"{hb}.{ln}.bias"].copy_(p[f"{b}/{ln}/bias"])
            for m in ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.out_proj", "mlp.fc1", "mlp.fc2"):
                sd[f"{hb}.{m}.weight"].copy_(p[f"{b}/{m.replace('.', '/')}/kernel"].t())
                sd[f"{hb}.{m}.bias"].copy_(p[f"{b}/{m.replace('.', '/')}/bias"])
    with torch.no_grad():
        sd["vision_model.embeddings.class_embedding"].copy_(pv["vision_model/embeddings/class_embedding"])
        sd["vision_model.embeddings.patch_embedding.weight"].copy_(
            pv["vision_model/embeddings/patch_embedding/kernel"].permute(3, 2, 0, 1))
        sd["vision_model.embeddings.position_embedding.weight"].copy_(pv["vision_model/embeddings/position_embedding/embedding"])
        for hf_n, fx in (("pre_layrnorm", "pre_layrnorm"), ("post_layernorm", "post_layernorm")):
            sd[f"vision_model.{hf_n}.weight"].copy_(pv[f"vision_model/{fx}/scale"])
            sd[f"vision_model.{hf_n}.bias"].copy_(pv[f"vision_model/{fx}/bias"])
        layers("vision_model", "vision_model", pv, vcfg.num_hidden_layers)
        sd["visual_projection.weight"].copy_(pv["visual_projection/kernel"].t())
        sd["text_model.embeddings.token_embedding.weight"].copy_(pt["text_model/embeddings/token_embedding/embedding"])
        sd["text_model.embeddings.position_embedding.weight"].copy_(pt["text_model/embeddings/position_embedding/embedding"])
        layers("text_model", "text_model", pt, tcfg.num_hidden_layers)
        sd["text_model.final_layer_norm.weight"].copy_(pt["text_model/final_layer_norm/scale"])
        sd["text_model.final_layer_norm.bias"].copy_(pt["text_model/final_layer_norm/bias"])
        sd["text_projection.weight"].copy_(model.text_projection.cpu().t())
    hf.load_state_dict(sd)
    return hf


PROMPTS = ["a cat", "two dogs playing in the snow", "a very small horse", ""]


def test_consistency_oracle_matches_transformers_clip_model(emu):
    model = CV.CLIPConsistency(CV.VIT_TINY, TINY_TEXT, device="cpu", seed=0)
    assert model.logit_scale == np.float32(2.6592)
    hf = _hf_clip_model(model)
    px = CV.preprocess(np.random.default_rng(4).integers(0, 256, (4, 64, 64, 3), dtype=np.uint8), 56)
    ids, _ = model.token_ids(PROMPTS)
    with torch.no_grad():
        out = hf(input_ids=torch.from_numpy(ids), pixel_values=torch.from_numpy(px).permute(0, 3, 1, 2))
    want = out.logits_per_image.diagonal()[:, None].numpy()
    np.testing.assert_allclose(_oracle_consistency(model, px, PROMPTS), want, rtol=1e-4, atol=1e-4)


def test_consistency_host_assembly_on_the_emulator(emu):
    model = CV.CLIPConsistency(CV.VIT_TINY, TINY_TEXT, device="cpu", seed=0)
    fn = C.callback_fns["consistency"](device="cpu", model=model)
    imgs = np.random.default_rng(5).random((4, 64, 64, 3)).astype(np.float32)
    s, info = fn(imgs, PROMPTS, {})
    assert s.dtype == np.float32 and s.shape == (4, 1) and info == {}
    # the reference formula on the emulated towers' own features
    u8 = torch.from_numpy((imgs * 255).astype(np.uint8))
    img = model.vision.image_features(torch.from_numpy(CV.preprocess((imgs * 255).astype(np.uint8), 56)))
    want = R.consistency(img.double().numpy(), model.text_features(PROMPTS).double().numpy(), np.float32(model.logit_scale))
    np.testing.assert_allclose(s, want, rtol=0, atol=1e-4)
    np.testing.assert_allclose(s, _oracle_consistency(model, CV.preprocess(u8.numpy(), 56), PROMPTS), atol=0.5)
    assert (fn(u8.numpy(), PROMPTS, {})[0] == s).all()


def test_consistency_refuses_prompts_longer_than_77_tokens(emu):
    model = CV.CLIPConsistency(CV.VIT_TINY, TINY_TEXT, device="cpu", seed=0)
    ids, pos = model.token_ids(["x" * 75])
    assert ids.shape == (1, 77) and pos[0] == 76 and ids[0, 76] == 49407
    with pytest.raises(ValueError, match="longer than 77"):
        model.token_ids(["a cat", "x" * 76])


# ------------------------------------------------------------------ registry and driver ----
REFERENCE_NAMES = {"vae", "aesthetic", "consistency", "jpeg", "neg_jpeg", "rotational", "rotational_corr", "mirror",
                   "mirror_corr", "thumbnail", "arange", "vqa", "llava_vqa", "llava_bertscore"}


def test_registry_has_every_reference_name():
    assert REFERENCE_NAMES <= set(C.callback_fns)
    for name in ("mirror", "mirror_corr", "rotational_corr"):
        assert C.callback_fns[name](device="cpu").accepts_uint8


@pytest.fixture()
def emulated_driver(emu, monkeypatch, tmp_path):
    from ddpo_b200 import unet as U, vae as V
    from ddpo_b200.diffusers_patch import pipeline_stable_diffusion as P, scheduling_ddim as SD
    from ddpo_b200.pipeline import policy_gradient as DRV
    from ddpo_b200.training import policy_gradient as PG
    E = emu
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
    # the full ViT-L/14 is the GPU tests' business: the dry run uses the tiny tower through the same host code
    monkeypatch.setitem(C.callback_fns, "rotational", functools.partial(C.rotational_symmetry_fn, cfg=CV.VIT_TINY))
    return E


@pytest.mark.parametrize("field", ["mirror", "rotational"])
def test_ddpo_epoch_driver_with_a_symmetry_reward(emulated_driver, field):
    from ddpo_b200 import utils
    from ddpo_b200.pipeline import policy_gradient as DRV
    models = utils.load_unet(None, pretrained_model="tiny", device="cpu", seed=0, text_encoder="stub")
    argv = ["--dataset", "compressed_animals", "--pretrained_model", "tiny", "--resolution", "128",
            "--sample_batch_size", "2", "--num_sample_batches_per_epoch", "2", "--n_inference_steps", "2",
            "--train_batch_size", "2", "--train_macro", "2", "--num_train_epochs", "1", "--save_freq", "100",
            "--savepath", f"run_{field}", "--seed", "3", "--filter_field", field]
    out = DRV.main(argv, models=models, max_epochs=1, save_last=False)
    rewards = np.asarray(out["history"][0]["rewards"]) if "rewards" in out["history"][0] else None
    assert len(out["history"]) == 1
    if rewards is not None:
        assert np.isfinite(rewards).all() and (rewards <= 0).all()
