"""GPU tests of the image-symmetry and consistency rewards (csrc/image_rewards.cu) on the H100: the bicubic resample
against Pillow byte for byte, the device preprocessing and the aesthetic scores against the host path bit for bit,
the pixel rewards against the NumPy restatement of the reference (tests/_rewards_ref.py), the CLIP-feature rewards
against the reference formula on the GPU towers' own features, the full-size towers against the fp32 oracle, argument
refusals, and one SD2-base 512 px DDPO epoch with ``--filter_field thumbnail``."""
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image, ImageOps

sys.path.insert(0, os.path.dirname(__file__))
import _rewards_ref as R  # noqa: E402

from ddpo_b200 import clip_vision as CV, ops  # noqa: E402
from ddpo_b200._lib import DdpoError  # noqa: E402
from ddpo_b200.training import callbacks as C  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
PIL_T = {CV.IDENTITY: lambda p: p, CV.MIRROR: ImageOps.mirror, CV.ROT90: lambda p: p.rotate(90),
         CV.ROT180: lambda p: p.rotate(180), CV.ROT270: lambda p: p.rotate(270)}
SIZES = [(512, 224), (512, 128), (512, 64), (512, 32), (128, 224), (64, 224), (32, 224), (256, 224), (768, 224),
         (224, 224)]


def _images(n, s, seed=0):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 256, (n, s, s, 3), dtype=np.uint8)
    a[1] = 0
    a[2] = np.where(rng.random((s, s, 3)) < 0.5, 0, 255)
    a[3, : s // 2] = 255
    return a


@pytest.mark.parametrize("src,dst", SIZES)
def test_resample_equals_pillow_byte_for_byte(src, dst):
    imgs = _images(8, src)
    dev = torch.from_numpy(imgs).to(DEV)
    for t, f in PIL_T.items():
        got = CV.resize_u8(dev, dst, dst, t)
        again = CV.resize_u8(dev, dst, dst, t)
        alone = CV.resize_u8(dev[5:6], dst, dst, t)
        torch.cuda.synchronize()
        want = np.stack([np.array(f(Image.fromarray(a)).resize((dst, dst), Image.BICUBIC)) for a in imgs])
        np.testing.assert_array_equal(got.cpu().numpy(), want, err_msg=f"transform {t}")
        assert torch.equal(got, again) and torch.equal(alone[0], got[5])


def test_normalised_pixels_and_aesthetic_scores_are_bit_identical_to_the_host_path():
    imgs = np.random.default_rng(1).random((8, 512, 512, 3)).astype(np.float32)
    u8 = torch.from_numpy(CV.to_uint8(imgs)).to(DEV)
    px = CV.preprocess_device(u8, 224)
    host = CV.preprocess(imgs, 224)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(px.cpu().numpy(), host)
    for t, f in PIL_T.items():
        want = CV.preprocess(np.stack([np.array(f(Image.fromarray(a))) for a in CV.to_uint8(imgs)]), 224)
        np.testing.assert_array_equal(CV.preprocess_device(u8, 224, t).cpu().numpy(), want)
    sc = CV.AestheticScorer(CV.VIT_L14, device=DEV, seed=0)
    got = sc(imgs, chunk=8)
    want = sc.score_features(sc.image_features(torch.from_numpy(host))).cpu().numpy()
    np.testing.assert_array_equal(got, want)


def test_pixel_rewards_equal_the_reference():
    imgs = np.random.default_rng(2).random((8, 512, 512, 3)).astype(np.float32)
    imgs[1] = (imgs[1] + imgs[1][:, ::-1]) / 2
    imgs[2] = (imgs[2] + np.rot90(imgs[2], 2)) / 2
    imgs[3] = 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        for name, ref in (("mirror", R.mirror), ("rotational_corr", R.rotational_corr)):
            s, _ = C.callback_fns[name]()(imgs, ["p"] * 8, {})
            assert s.dtype == np.float64 and s.shape == (8,)
            assert (s == ref(imgs)).all(), name
        s, _ = C.callback_fns["mirror_corr"]()(imgs, ["p"] * 8, {})
        want = R.mirror_corr(imgs, np.float64)
    assert s.dtype == np.float32 and s.shape == (8,) and np.isnan(s[3]) and np.isnan(want[3])
    np.testing.assert_allclose(np.delete(s, 3), np.delete(want, 3), rtol=0, atol=1e-6)


def _features_fn(tower):
    def f(px):
        out = tower.image_features(torch.from_numpy(np.ascontiguousarray(px)))
        return out.cpu().numpy()
    return f


@pytest.mark.parametrize("name,ref", [("rotational", R.rotational), ("thumbnail", R.thumbnail)])
def test_angle_rewards_match_the_reference_formula_on_the_towers_features(name, ref):
    imgs = np.random.default_rng(3).random((8, 512, 512, 3)).astype(np.float32)
    fn = C.callback_fns[name]()
    s, info = fn(imgs, ["p"] * 8, {})
    assert s.dtype == np.float32 and s.shape == (8,) and info == {}
    tower = CV.CLIPImageTower(CV.VIT_L14, device=DEV, seed=0)
    want = ref(imgs, _features_fn(tower), 224)
    np.testing.assert_allclose(s, want, rtol=0, atol=1e-4)
    assert (fn((imgs * 255).astype(np.uint8), ["p"] * 8, {})[0] == s).all()


def test_consistency_matches_the_reference_formula_on_the_towers_features():
    prompts = ["a cat", "a dog", "two horses in a field", "a small bird", "fish", "", "an owl at night", "a llama"]
    imgs = np.random.default_rng(4).random((8, 512, 512, 3)).astype(np.float32)
    model = CV.CLIPConsistency(device=DEV, seed=0)
    s, info = C.callback_fns["consistency"](model=model)(imgs, prompts, {})
    assert s.dtype == np.float32 and s.shape == (8, 1)
    img = model.vision.image_features(torch.from_numpy(CV.preprocess(imgs, 224))).cpu().double().numpy()
    txt = model.text_features(prompts).cpu().double().numpy()
    np.testing.assert_allclose(s, R.consistency(img, txt, np.float32(model.logit_scale)), rtol=0, atol=1e-4)


@pytest.mark.parametrize("cfg_name", ["VIT_L14", "VIT_B32"])
def test_full_size_towers_against_the_fp32_oracle(cfg_name):
    from oracle import clip_vision as OCV
    cfg = getattr(CV, cfg_name)
    tower = CV.CLIPImageTower(cfg, device=DEV, seed=0)
    px = torch.from_numpy(CV.preprocess(np.random.default_rng(5).random((4, 512, 512, 3)).astype(np.float32), 224))
    got = tower.image_features(px).cpu()
    want = OCV.image_features(CV.views(tower.params.cpu(), cfg, head=False), cfg, px)
    rel = ((got - want).norm() / want.norm()).item()
    print(f"{cfg_name} image features vs fp32 oracle: relative L2 error {rel:.3e} ({torch.cuda.get_device_name()})")
    assert rel < 2e-2, rel


def test_argument_refusals_write_nothing():
    src = torch.randint(0, 256, (2, 60, 90, 3), dtype=torch.uint8, device=DEV)
    dst = torch.full((2, 90, 32, 3), 7, dtype=torch.uint8, device=DEV)
    t = CV.resample_table(60, 32)
    td = torch.from_numpy(t.copy()).to(DEV)
    with pytest.raises(DdpoError, match="square"):
        ops.resample_u8(src, CV.ROT90, 0, t, td, dst)
    bad = t.copy()
    bad[3, 0] = 89                                          # a window past the input's end
    with pytest.raises(DdpoError, match="outside"):
        ops.resample_u8(src, CV.IDENTITY, 0, bad, td, torch.full((2, 60, 32, 3), 7, dtype=torch.uint8, device=DEV))
    out = torch.full((2, 32, 32, 3), 7.0, device=DEV)
    with pytest.raises(DdpoError):
        ops.clip_normalize_u8(src, 40, 0, out)
    st = torch.full((2, 4), 7, dtype=torch.int64, device=DEV)
    with pytest.raises(DdpoError):
        ops.pair_stats_u8(src, CV.ROT90, st)
    ang = torch.full((2,), 7.0, device=DEV)
    with pytest.raises(DdpoError):
        ops.feature_angles(torch.zeros(2, 8, device=DEV), 1, ang)
    torch.cuda.synchronize()
    assert (dst == 7).all() and (out == 7).all() and (st == 7).all() and (ang == 7).all()


def test_ddpo_epoch_sd2_base_thumbnail(tmp_path, monkeypatch):
    from ddpo_b200 import utils
    from ddpo_b200.pipeline import policy_gradient as PG
    from ddpo_b200.training import policy_gradient as pg
    monkeypatch.chdir(tmp_path)
    monkeypatch.setenv(utils.serialization.ALLOW_RANDOM_ENV, "1")
    pg._GRAPHS.clear()
    model = "random:stabilityai/stable-diffusion-2-base"
    models = utils.load_unet(None, pretrained_model=model, device="cuda", seed=0)
    argv = ["--dataset", "compressed_animals", "--pretrained_model", model, "--resolution", "512",
            "--sample_batch_size", "2", "--num_sample_batches_per_epoch", "1", "--n_inference_steps", "4",
            "--train_batch_size", "1", "--train_macro", "2", "--num_train_epochs", "1", "--save_freq", "100",
            "--learning_rate", "1e-5", "--savepath", "thumb", "--seed", "3", "--filter_field", "thumbnail"]
    out = PG.main(argv, models=models, max_epochs=1, save_last=False)
    r = out["history"][0]["mean_reward"]
    assert np.isfinite(r) and r <= 0
    pg._GRAPHS.clear()
