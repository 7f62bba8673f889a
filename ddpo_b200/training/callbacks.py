"""Reward callbacks -- mirrors the registry/signature of ``ddpo/training/callbacks.py:540-564``:
``callback_fns[name]() -> fn(images f32 NHWC in [0,1] [N,H,W,3], prompts, metadata) -> (scores, info)``.
``jpeg`` / ``neg_jpeg`` (:143-163, JPEG q=95 size in kB via PIL, ``hdf5.py:25-37``) and ``arange`` (:347-354)
are real; the model-based rewards (aesthetic CLIP+MLP, LLaVA over HTTP) need weights / a server that do not
exist offline and are provided as cached-score stubs (BASELINE.json configs 3 and 5).  The image-symmetry rewards
(``mirror``, ``mirror_corr``, ``rotational``, ``rotational_corr``, ``thumbnail``, :166-344) and ``consistency``
(:122-140) run on the GPU kernels: the images go to the device once as uint8 and every transform, resample and reduction
happens there (``csrc/image_rewards.cu``); their CLIP towers are random-init, seeded as ``aesthetic``'s."""
import io
import random

import numpy as np
import torch

from .. import clip_vision as CV, ops


def encode_jpeg(x, quality=95):
    from PIL import Image
    x = np.asarray(x)
    if np.issubdtype(x.dtype, np.floating):
        assert np.abs(x).max() <= 1.0
        x = (x * 255).astype(np.uint8)
    buf = io.BytesIO()
    Image.fromarray(x).save(buf, "JPEG", quality=quality)
    return np.frombuffer(buf.getvalue(), dtype=np.uint8)


def jpeg_fn(devices=None, jit=False):
    assert not jit

    def _fn(images, prompts, metadata):
        sizes_kb = [len(encode_jpeg(im)) / 1000.0 for im in images]
        return -np.array(sizes_kb)[:, None], {}
    _fn.accepts_uint8 = True   # encode_jpeg takes the bytes as they are: the driver converts on the device (4x fewer D2H bytes)
    return _fn


def neg_jpeg_fn(*args, **kwargs):
    inner = jpeg_fn(*args, **kwargs)

    def _fn(*a, **k):
        scores, info = inner(*a, **k)
        return -scores, info
    _fn.accepts_uint8 = True
    return _fn


def arange_fn(devices=None, jit=False):
    def _fn(images, prompts, metadata):
        return np.arange(len(images)), {}
    _fn.accepts_uint8 = True
    return _fn


ALLOW_STUB_ENV = "DDPO_ALLOW_STUB_REWARDS"


def _cached_score_stub(name, shape_2d):
    """Stand-in for a reward MODEL that cannot exist offline (weights / server): N(0,1) scores keyed by the prompts,
    INDEPENDENT OF THE IMAGES.  Optimising it optimises noise, so instantiating one is an error unless the caller opts in
    with ``$DDPO_ALLOW_STUB_REWARDS=1`` (benchmarks and tests of the plumbing do)."""
    def factory(devices=None, jit=False):
        import os
        if os.environ.get(ALLOW_STUB_ENV) != "1":
            raise RuntimeError(
                f"reward '{name}' needs a model that is not available here (LLaVA server / CLIP weights); the only "
                f"offline substitute is a cached-score stub that ignores the images.  Set {ALLOW_STUB_ENV}=1 to accept "
                f"it explicitly, point $DDPO_LLAVA_URL at a server, or set $DDPO_AESTHETIC_GPU=1 for the GPU aesthetic tower.")
        import warnings
        warnings.warn(f"reward '{name}' is a cached-score STUB: scores do not depend on the images", RuntimeWarning)

        def _fn(images, prompts, metadata):
            import hashlib
            digest = hashlib.sha1("\x1f".join([name] + [str(p) for p in prompts]).encode()).hexdigest()
            rng = np.random.default_rng(int(digest, 16) % (2 ** 32))   # reproducible across processes and runs
            s = rng.standard_normal(len(images)).astype(np.float32)
            return (s[:, None] if shape_2d else s), {"stub": True}
        return _fn
    return factory


AESTHETIC_GPU_ENV = "DDPO_AESTHETIC_GPU"


def aesthetic_fn(devices=None, rng=0, cache="cache", jit=True):
    """Reference ``callbacks.py:60-95``: CLIP ViT-L/14 image features -> L2 normalise -> LAION aesthetic head; returns
    ``[N, 1]`` scores.  The model runs on the GPU kernels (``ddpo_b200/clip_vision.py``: CLIP ViT-L/14 image tower +
    LAION head; weights are random-init unless a checkpoint is found -- none exists offline -- and the LAION head is read
    from ``cache/`` when that file exists).  ``$DDPO_AESTHETIC_GPU=0`` (or no CUDA device) selects the cached-score stub,
    which itself needs ``$DDPO_ALLOW_STUB_REWARDS=1``."""
    import os
    import torch
    want_gpu = os.environ.get(AESTHETIC_GPU_ENV, "1") == "1" and torch.cuda.is_available()
    if not want_gpu:
        return _cached_score_stub("aesthetic", True)(devices, jit)
    from ..clip_vision import AestheticScorer
    scorer = AestheticScorer(seed=int(rng), cache=cache)

    def _wrapper(images, prompts, metadata):
        del prompts, metadata
        return scorer(images), {}
    return _wrapper


LLAVA_URL_ENV = "DDPO_LLAVA_URL"   # e.g. http://127.0.0.1:8085 (the reference hard-codes this address, callbacks.py:470)


def llava_bertscore_fn(devices=None, jit=False, url=None, batch_size=16, timeout=120):
    """Reference ``callbacks.py:464-537``: the alignment reward is computed by a LLaVA + BERTScore server spoken to with
    pickle-over-HTTP.  Wire format kept byte for byte: POST body = ``pickle.dumps({"images": [JPEG q=80 bytes],
    "queries": [["Answer concisely: what is going on in this image?"]] * n, "answers": [[f"The image contains {p}"]]})``
    in batches of 16; response = pickle of ``{"recall", "precision", "f1", "outputs"}``; the reward is the recall.
    Without a server (``url`` / ``$DDPO_LLAVA_URL`` unset -- the offline default, BASELINE config 5 "reward server stubbed
    to cached scores") the cached-score stub answers instead."""
    import os
    url = url or os.environ.get(LLAVA_URL_ENV)
    if not url:
        return _cached_score_stub("llava_bertscore", False)(devices, jit)
    import pickle
    from io import BytesIO

    import requests
    from PIL import Image
    from requests.adapters import HTTPAdapter, Retry
    sess = requests.Session()
    sess.mount("http://", HTTPAdapter(max_retries=Retry(total=1000, backoff_factor=1, status_forcelist=[500],
                                                        allowed_methods=False)))

    def _fn(images, prompts, metadata):
        del metadata
        images = (np.asarray(images) * 255).astype(np.uint8)
        n_batches = int(np.ceil(len(images) / batch_size))
        all_scores, all_info = [], {"precision": [], "f1": [], "outputs": []}
        for image_batch, prompt_batch in zip(np.array_split(images, n_batches), np.array_split(np.asarray(prompts), n_batches)):
            jpeg_images = []
            for image in image_batch:
                buffer = BytesIO()
                Image.fromarray(image).save(buffer, format="JPEG", quality=80)
                jpeg_images.append(buffer.getvalue())
            data = {"images": jpeg_images,
                    "queries": [["Answer concisely: what is going on in this image?"]] * len(image_batch),
                    "answers": [[f"The image contains {prompt}"] for prompt in prompt_batch]}
            response = sess.post(url, data=pickle.dumps(data), timeout=timeout)
            response_data = pickle.loads(response.content)
            all_scores += np.array(response_data["recall"]).reshape(-1).tolist()
            all_info["precision"] += np.array(response_data["precision"]).reshape(-1).tolist()
            all_info["f1"] += np.array(response_data["f1"]).reshape(-1).tolist()
            all_info["outputs"] += np.array(response_data["outputs"]).reshape(-1).tolist()
        return np.array(all_scores), {k: np.array(v) for k, v in all_info.items()}
    return _fn


def vae_fn(devices=None, dtype="float32", jit=True, encoder=None, pretrained_model="tiny", seed=0, device="cuda"):
    """Reference ``callbacks.py:37-57``: ``fn(images NHWC in [0, 1]) -> (concatenate([posterior mean, logvar], -1), {})``,
    the ``"vae"`` field of the RWR shards.  ``encoder``: a ``ddpo_b200.vae.VAEEncoder`` (``utils.load_unet`` attaches the
    checkpoint's, or a random-init one, as ``pipeline.vae_encoder``); without one an encoder of ``pretrained_model``'s
    architecture is built with random-init weights."""
    if encoder is None:
        from ..vae import VAEEncoder, vae_config_for
        encoder = VAEEncoder(vae_config_for(pretrained_model), device=device, seed=seed)

    def _fn(images, prompts=None, metadata=None):
        import torch
        mom = encoder.encode(torch.as_tensor(np.asarray(images, np.float32)))
        return mom.float().cpu().numpy(), {}
    return _fn


def _device(device=None):
    if device is not None:
        return torch.device(device)
    return torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")


def _image_bytes(images, device):
    """the reference's ``(image * 255).astype(np.uint8)`` (:181) for float images, uint8 as it is; one copy to the device"""
    x = np.asarray(images)
    if x.dtype != np.uint8:
        x = (x * 255).astype(np.uint8)
    assert x.ndim == 4 and x.shape[-1] == 3, x.shape
    return torch.from_numpy(np.ascontiguousarray(x)).to(device)


def _pair_stats(images, transform, device):
    """per image, exact integer sums against its mirror / 180-degree rotation: uint64 [N, 4] (wrapped squared difference,
    sum a, sum a^2, sum a T(a)) and the number of bytes per image"""
    u8 = _image_bytes(images, device)
    st = torch.empty(len(u8), 4, dtype=torch.int64, device=device)
    ops.pair_stats_u8(u8, transform, st)
    return st.cpu().numpy().view(np.uint64), u8[0].numel()


def _wrapped_mse(images, transform, device):
    """``((a - T a) ** 2).mean(axis=(1, 2, 3))`` of uint8 arrays, numpy's uint8 wrap included: the float64 mean of
    integers below 2**53 is exactly their sum over the count"""
    st, n = _pair_stats(images, transform, device)
    return st[:, 0].astype(np.float64) / n


def mirror_symmetry_fn(devices=None, jit=False, device=None):
    """Reference :244-260: ``-((pils - mirrored) ** 2).mean(axis=(1, 2, 3))`` on uint8 arrays, float64 [N].  The
    subtraction and the square wrap modulo 256, as numpy's uint8 arithmetic does in the reference."""
    dev = _device(device)

    def _fn(images, prompts, metadata):
        return -_wrapped_mse(images, CV.MIRROR, dev), {}
    _fn.accepts_uint8 = True
    return _fn


def rotational_correlation_fn(devices=None, jit=False, device=None):
    """Reference :216-241: the same wrapped mean squared difference against ``pil.rotate(180)``, negated; float64 [N]."""
    dev = _device(device)

    def _fn(images, prompts, metadata):
        return -_wrapped_mse(images, CV.ROT180, dev), {}
    _fn.accepts_uint8 = True
    return _fn


def mirror_correlation_fn(devices=None, jit=False, device=None):
    """Reference :268-292: minus the Pearson correlation of an image's bytes with its mirror's, float32 [N].  Computed
    exactly from integer sums (the reference's float32 cov differs from it by ~1e-7).  An image of zero variance (a flat
    image, e.g. all black) scores NaN, as 0 / 0 does in the reference."""
    dev = _device(device)

    def _fn(images, prompts, metadata):
        st, n = _pair_stats(images, CV.MIRROR, dev)
        out = np.empty(len(st), np.float32)
        for i, (_, sa, saa, sab) in enumerate(st.tolist()):
            den = n * saa - sa * sa          # the mirror is a permutation: sum b = sum a, sum b^2 = sum a^2
            out[i] = np.nan if den == 0 else -(n * sab - sa * sa) / den
        return out, {}
    _fn.accepts_uint8 = True
    return _fn


def _angle_reward(variants, images, device):
    """-mean over variants >= 1 of the angle (degrees) between the CLIP features of variant 0 and variant v (reference
    :196-211, :327-342); ``variants`` are functions of the uint8 device batch to the tower's feature rows"""
    u8 = _image_bytes(images, device)
    feats = torch.cat([v(u8) for v in variants])
    out = torch.empty(len(u8), dtype=torch.float32, device=device)
    ops.feature_angles(feats, len(variants), out)
    return -out.cpu().numpy(), {}


def rotational_symmetry_fn(devices=None, jit=True, rng=0, cfg=None, device=None):
    """Reference :166-213: CLIP ViT-L/14 features of ``pil.rotate(0 / 90 / 180 / 270)``, minus the mean angle between
    the original's and each rotation's; float32 [N].  Square images only (Pillow rotates others through its affine path)."""
    dev = _device(device)
    tower = CV.CLIPImageTower(cfg or CV.VIT_L14, device=dev, seed=int(rng))
    variants = [lambda u8, t=t: tower.features(u8, t) for t in (CV.IDENTITY, CV.ROT90, CV.ROT180, CV.ROT270)]

    def _fn(images, prompts, metadata):
        return _angle_reward(variants, images, dev)
    _fn.accepts_uint8 = True
    return _fn


def thumbnail_fn(devices=None, jit=True, rng=0, cfg=None, device=None):
    """Reference :295-344: CLIP ViT-L/14 features of the image and of its bicubic thumbnails at 1/4, 1/8 and 1/16 size
    (``pil.resize``), minus the mean angle between the original's and each thumbnail's; float32 [N]."""
    dev = _device(device)
    tower = CV.CLIPImageTower(cfg or CV.VIT_L14, device=dev, seed=int(rng))

    def thumb(d):
        return lambda u8: tower.features(CV.resize_u8(u8, u8.shape[2] // d, u8.shape[1] // d))
    variants = [tower.features] + [thumb(d) for d in (4, 8, 16)]

    def _fn(images, prompts, metadata):
        return _angle_reward(variants, images, dev)
    _fn.accepts_uint8 = True
    return _fn


def consistency_fn(devices=None, jit=False, rng=0, model=None, device=None):
    """Reference :122-140: CLIP ViT-B/32 ``logits_per_image.diagonal()[:, None]`` of each image with its own prompt,
    float32 [N, 1] (``clip_vision.CLIPConsistency``)."""
    dev = _device(device)
    model = model or CV.CLIPConsistency(device=dev, seed=int(rng))

    def _fn(images, prompts, metadata):
        return model(_image_bytes(images, dev), prompts)[:, None], {}
    _fn.accepts_uint8 = True
    return _fn


def evaluate_callbacks(fns, images, prompts, metadata):
    if type(prompts[0]) == list:
        prompts = [random.choice(p) for p in prompts]
    images = np.asarray(images)
    if images.dtype != np.uint8:   # uint8: the driver already applied the rewards' own cast on the device
        images = images.astype(np.float32)
    return {key: fn(images, prompts, metadata) for key, fn in fns.items()}


callback_fns = {
    "jpeg": jpeg_fn,
    "neg_jpeg": neg_jpeg_fn,
    "arange": arange_fn,
    "aesthetic": aesthetic_fn,
    "llava_bertscore": llava_bertscore_fn,
    "llava_vqa": _cached_score_stub("llava_vqa", False),     # callbacks.py:401-461 needs the LLaVA server; offline stub
    "vqa": _cached_score_stub("vqa", True),
    "vae": vae_fn,
    "consistency": consistency_fn,
    "rotational": rotational_symmetry_fn,
    "rotational_corr": rotational_correlation_fn,
    "mirror": mirror_symmetry_fn,
    "mirror_corr": mirror_correlation_fn,
    "thumbnail": thumbnail_fn,
}
