"""Aesthetic reward model on the libddpo_b200 kernels -- what the reference builds in ``aesthetic_fn``
(``ddpo/training/callbacks.py:60-95``): ``FlaxCLIPModel.get_image_features`` of CLIP ViT-L/14 (3P transformers==4.28.1:
patch embedding, class + position embeddings, pre-LayerNorm, 24 pre-LN transformer layers with ``quick_gelu``,
post-LayerNorm of the CLS token, visual projection 1024 -> 768), L2 normalisation, and the LAION ``AestheticClassifier``
(``ddpo/models/laion.py:7-18``: five Dense layers 768-1024-128-64-16-1 without activations; dropout is deterministic).

The oracle (``oracle/clip_vision.py``) is pinned against the installed ``transformers`` ``CLIPVisionModelWithProjection``;
the CUDA path (``csrc/vision.cu`` + the text tower's building blocks) agrees with it within 2e-2 relative on the GPU
(``tests/test_gpu_zz_grouped_temb_aesthetic.py``; full-size ViT-L/14 run included).  Weights are random-init (no checkpoints offline); the
LAION head loads ``sac+logos+ava1-l14-linearMSE.pth`` from ``cache/`` when the file exists, as the reference does.

The same image tower (``CLIPImageTower``) serves the image-symmetry rewards (``rotational``, ``thumbnail``) and, at
ViT-B/32 size with the CLIP text tower, the ``consistency`` reward (``CLIPConsistency``).  Their pixels are prepared on
the device (``preprocess_device``: PIL-exact bicubic resample of a mirrored or rotated source, centre crop, CLIP
normalisation; ``csrc/image_rewards.cu``), bit-identical to the host ``preprocess``, which stays as the reference.
"""
import functools
import os
from dataclasses import dataclass
from typing import Dict, List, Tuple

import numpy as np
import torch

from . import ops
from .unet import Arena

BF16, F32 = torch.bfloat16, torch.float32
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
HEAD_SIZES = (1024, 128, 64, 16, 1)


@dataclass(frozen=True)
class CLIPVisionConfig:
    image_size: int = 224
    patch_size: int = 14
    hidden_size: int = 1024
    intermediate_size: int = 4096
    num_hidden_layers: int = 24
    num_attention_heads: int = 16
    projection_dim: int = 768
    hidden_act: str = "quick_gelu"
    layer_norm_eps: float = 1e-5

    @property
    def n_patches(self):
        return (self.image_size // self.patch_size) ** 2


VIT_L14 = CLIPVisionConfig()
VIT_B32 = CLIPVisionConfig(patch_size=32, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                           num_attention_heads=12, projection_dim=512)
VIT_TINY = CLIPVisionConfig(image_size=56, patch_size=14, hidden_size=128, intermediate_size=256, num_hidden_layers=2,
                            num_attention_heads=2, projection_dim=64)


def param_manifest(cfg: CLIPVisionConfig, head: bool = True) -> List[Tuple[str, Tuple[int, ...]]]:
    """the image tower, then (``head``) the LAION aesthetic head"""
    D, I, P = cfg.hidden_size, cfg.intermediate_size, cfg.patch_size
    out = [("vision_model/embeddings/class_embedding", (D,)),
           ("vision_model/embeddings/patch_embedding/kernel", (P, P, 3, D)),
           ("vision_model/embeddings/position_embedding/embedding", (cfg.n_patches + 1, D)),
           ("vision_model/pre_layrnorm/scale", (D,)), ("vision_model/pre_layrnorm/bias", (D,))]
    for i in range(cfg.num_hidden_layers):
        b = f"vision_model/encoder/layers/{i}"
        out += [(f"{b}/layer_norm1/scale", (D,)), (f"{b}/layer_norm1/bias", (D,))]
        for p in ("q_proj", "k_proj", "v_proj", "out_proj"):
            out += [(f"{b}/self_attn/{p}/kernel", (D, D)), (f"{b}/self_attn/{p}/bias", (D,))]
        out += [(f"{b}/layer_norm2/scale", (D,)), (f"{b}/layer_norm2/bias", (D,)),
                (f"{b}/mlp/fc1/kernel", (D, I)), (f"{b}/mlp/fc1/bias", (I,)),
                (f"{b}/mlp/fc2/kernel", (I, D)), (f"{b}/mlp/fc2/bias", (D,))]
    out += [("vision_model/post_layernorm/scale", (D,)), ("vision_model/post_layernorm/bias", (D,)),
            ("visual_projection/kernel", (D, cfg.projection_dim))]
    if not head:
        return out
    k = cfg.projection_dim
    for i, n in enumerate(HEAD_SIZES):     # AestheticClassifier: Dense_0 .. Dense_4
        out += [(f"aesthetic/Dense_{i}/kernel", (k, n)), (f"aesthetic/Dense_{i}/bias", (n,))]
        k = n
    return out


def param_offsets(cfg: CLIPVisionConfig, align: int = 64, head: bool = True):
    off, table = 0, {}
    for name, shape in param_manifest(cfg, head):
        table[name] = (off, shape)
        off += (int(np.prod(shape)) + align - 1) // align * align
    return table, off


def num_params(cfg: CLIPVisionConfig, head: bool = False) -> int:
    return sum(int(np.prod(s)) for n, s in param_manifest(cfg) if head or not n.startswith("aesthetic/"))


def init_flat_params(cfg: CLIPVisionConfig, seed: int = 0, head: bool = True) -> torch.Tensor:
    """the tower's draws come first, so a tower without the head gets the same weights as one with it"""
    table, total = param_offsets(cfg, head=head)
    g = torch.Generator(device="cpu").manual_seed(seed)
    flat = torch.zeros(total, dtype=torch.float32)
    for name, (off, shape) in table.items():
        n = int(np.prod(shape))
        leaf = name.rsplit("/", 1)[1]
        if leaf == "kernel":
            v = torch.randn(n, generator=g) / np.sqrt(int(np.prod(shape[:-1])))
        elif leaf in ("embedding", "class_embedding"):
            v = 0.5 * torch.randn(n, generator=g)
        elif leaf == "scale":
            v = 1.0 + 0.1 * torch.randn(n, generator=g)
        else:
            v = 0.02 * torch.randn(n, generator=g)
        flat[off:off + n] = v
    return flat


def views(flat: torch.Tensor, cfg: CLIPVisionConfig, head: bool = True) -> Dict[str, torch.Tensor]:
    table, _ = param_offsets(cfg, head=head)
    return {k: flat[o:o + int(np.prod(s))].view(*s) for k, (o, s) in table.items()}


def preprocess(images, size):
    """``CLIPProcessor(images=list(images))`` for square float images in [0,1]: uint8 -> bicubic resize to ``size`` ->
    rescale -> normalise; returns float32 NHWC (the kernels' layout)."""
    from PIL import Image
    out = np.empty((len(images), size, size, 3), np.float32)
    for i, im in enumerate(images):
        im = np.asarray(im)
        if np.issubdtype(im.dtype, np.floating):
            im = (np.clip(im, 0, 1) * 255).astype(np.uint8)
        pil = Image.fromarray(im)
        if pil.size != (size, size):
            w, h = pil.size
            s = size / min(w, h)                                  # shortest edge to `size`, then centre crop
            pil = pil.resize((max(size, round(w * s)), max(size, round(h * s))), Image.BICUBIC)
            l, t = (pil.size[0] - size) // 2, (pil.size[1] - size) // 2
            pil = pil.crop((l, t, l + size, t + size))
        out[i] = (np.asarray(pil, np.float32) / 255.0 - CLIP_MEAN) / CLIP_STD
    return out


# source transforms of preprocess_device (include/ddpo_b200.h DDPO_IMAGE_*): ImageOps.mirror and Image.rotate's
# transposes.  rotate(90) turns counter-clockwise, as np.rot90(a, 1) does.
IDENTITY, MIRROR, ROT90, ROT180, ROT270 = range(5)


def _bicubic(x):
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


@functools.lru_cache(maxsize=None)
def resample_table(n_in: int, n_out: int) -> np.ndarray:
    """Pillow's ``precompute_coeffs`` for BICUBIC (``Resample.c``), in double as Pillow computes it, with its 22-bit
    rounding of each weight away from zero: int32 [n_out, 2 + ksize] rows of (xmin, n, n weights, zero padding)."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support, ss = 2.0 * fs, 1.0 / fs
    rows = []
    for i in range(n_out):
        center = (i + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), n_in) - xmin
        w = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(n)]
        tot = 0.0
        for v in w:
            tot += v
        if tot != 0.0:
            w = [v / tot for v in w]
        rows.append([xmin, n] + [int(v * (1 << 22) + (0.5 if v >= 0 else -0.5)) for v in w])
    ksize = max(len(r) for r in rows) - 2
    table = np.zeros((n_out, 2 + ksize), np.int32)
    for i, r in enumerate(rows):
        table[i, :len(r)] = r
    table.setflags(write=False)
    return table


_DEVICE_TABLES: Dict[Tuple[int, int, str], torch.Tensor] = {}


def _resample(src, transform, axis, n_out, dst):
    h, w = src.shape[1:3]
    n_in = (w if transform in (IDENTITY, MIRROR, ROT180) else h) if axis == 0 else \
           (h if transform in (IDENTITY, MIRROR, ROT180) else w)
    table = resample_table(int(n_in), int(n_out))
    key = (int(n_in), int(n_out), str(src.device))
    if key not in _DEVICE_TABLES:
        _DEVICE_TABLES[key] = torch.from_numpy(table.copy()).to(src.device)
    ops.resample_u8(src, transform, axis, table, _DEVICE_TABLES[key], dst)


def resize_u8(src, width: int, height: int, transform: int = IDENTITY):
    """``Image.resize((width, height), BICUBIC)`` of ``transform(image)`` for a uint8 NHWC batch on the device, as
    Pillow runs it: the width pass first (stored as uint8), then the height pass; a pass whose size does not change is
    skipped, and a transform with no resize is one identity-weight pass."""
    B, h, w, _ = src.shape
    th, tw = (w, h) if transform in (ROT90, ROT270) else (h, w)
    do_w, do_h = tw != width, th != height
    if not do_h:
        do_w = True
    cur = src
    if do_w:
        cur = torch.empty(B, th, width, 3, dtype=torch.uint8, device=src.device)
        _resample(src, transform, 0, width, cur)
        transform = IDENTITY
    if do_h:
        out = torch.empty(B, height, width, 3, dtype=torch.uint8, device=src.device)
        _resample(cur, transform, 1, height, out)
        cur = out
    return cur


def to_uint8(images):
    """host images -> uint8 NHWC numpy: uint8 as it is, float through the reference's ``(x * 255).astype(uint8)``
    (clipped to [0, 1] first, as ``preprocess`` does)"""
    x = np.asarray(images)
    if np.issubdtype(x.dtype, np.floating):
        x = (np.clip(x, 0, 1) * 255).astype(np.uint8)
    assert x.dtype == np.uint8 and x.ndim == 4 and x.shape[-1] == 3, (x.dtype, x.shape)
    return np.ascontiguousarray(x)


def preprocess_device(images_u8, size: int, transform: int = IDENTITY) -> torch.Tensor:
    """``preprocess`` of ``transform(image)`` on the device, bit-identical to it: uint8 NHWC device batch -> shortest
    edge to ``size`` (bicubic), centre crop, CLIP normalisation -> fp32 NHWC [B, size, size, 3]."""
    B, h, w, _ = images_u8.shape
    if transform in (ROT90, ROT270):
        h, w = w, h
    if (w, h) != (size, size):
        s = size / min(w, h)
        w, h = max(size, round(w * s)), max(size, round(h * s))
    u8 = images_u8 if (transform == IDENTITY and (w, h) == tuple(images_u8.shape[2:0:-1])) else \
        resize_u8(images_u8, w, h, transform)
    out = torch.empty(B, size, size, 3, dtype=F32, device=images_u8.device)
    ops.clip_normalize_u8(u8, (h - size) // 2, (w - size) // 2, out)
    return out


class CLIPImageTower:
    """``get_image_features`` of a CLIP vision tower (``FlaxCLIPModel``) on the kernels; parameters laid out by
    ``param_offsets(cfg, head=self.HEAD)``."""
    HEAD = False

    def __init__(self, cfg: CLIPVisionConfig = VIT_L14, flat_params: torch.Tensor = None, device="cuda", seed: int = 0):
        assert cfg.hidden_size % 64 == 0 and cfg.hidden_size // cfg.num_attention_heads == 64, "head width must be 64"
        assert cfg.projection_dim % 32 == 0 and cfg.intermediate_size % 64 == 0
        self.cfg = cfg
        self.device = torch.device(device)
        self.table, self.total = param_offsets(cfg, head=self.HEAD)
        if flat_params is None:
            flat_params = init_flat_params(cfg, seed, head=self.HEAD)
        assert flat_params.numel() == self.total
        self.params = flat_params.to(self.device, F32).contiguous()
        self.arena = Arena(self.device)
        self.kpad = (cfg.patch_size * cfg.patch_size * 3 + 63) // 64 * 64
        self.w: Dict[str, torch.Tensor] = {}
        self.qkv_bias: Dict[str, torch.Tensor] = {}
        self.refresh_weights()

    def p(self, name):
        off, shape = self.table[name]
        return self.params[off:off + int(np.prod(shape))].view(*shape)

    def refresh_weights(self):
        cfg = self.cfg
        D, I = cfg.hidden_size, cfg.intermediate_size
        k = cfg.patch_size * cfg.patch_size * 3
        self.w["patch"] = torch.zeros(D, self.kpad, dtype=BF16, device=self.device)     # zero K padding
        ops.prep_weight(self.p("vision_model/embeddings/patch_embedding/kernel"), self.w["patch"], k, D, ldk=self.kpad)
        for i in range(cfg.num_hidden_layers):
            b = f"vision_model/encoder/layers/{i}"
            key = b + "/self_attn/qkv"
            self.w[key] = torch.empty(3 * D, D, dtype=BF16, device=self.device)
            self.qkv_bias[key] = torch.empty(3 * D, dtype=F32, device=self.device)
            for j, pn in enumerate(("q_proj", "k_proj", "v_proj")):
                ops.prep_weight(self.p(f"{b}/self_attn/{pn}/kernel"), self.w[key], D, D, row_offset=j * D)
                self.qkv_bias[key][j * D:(j + 1) * D].copy_(self.p(f"{b}/self_attn/{pn}/bias"))
            for name, kk, n in ((b + "/self_attn/out_proj", D, D), (b + "/mlp/fc1", D, I), (b + "/mlp/fc2", I, D)):
                self.w[name] = torch.empty(n, kk, dtype=BF16, device=self.device)
                ops.prep_weight(self.p(name + "/kernel"), self.w[name], kk, n)
        self.w["proj"] = torch.empty(cfg.projection_dim, D, dtype=BF16, device=self.device)
        ops.prep_weight(self.p("visual_projection/kernel"), self.w["proj"], D, cfg.projection_dim)

    @torch.no_grad()
    def image_features(self, pixel_values_nhwc: torch.Tensor) -> torch.Tensor:
        """normalised pixels fp32 NHWC [B, S, S, 3] -> ``get_image_features`` [B, projection_dim] fp32"""
        cfg, A = self.cfg, self.arena
        x_img = pixel_values_nhwc.to(self.device, F32).contiguous()
        B = x_img.shape[0]
        assert tuple(x_img.shape[1:]) == (cfg.image_size, cfg.image_size, 3)
        D, I, H, N = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads, cfg.n_patches
        L = N + 1
        m = B * L
        patches = A.alloc((B * N, self.kpad), BF16)
        ops.patchify_bf16(x_img, patches, cfg.patch_size)
        pe = A.alloc((B * N, D), F32)
        ops.igemm(a0=patches, wt=self.w["patch"], n=D, c0=self.kpad, m=B * N, out_f32=pe)
        tok = A.alloc((m, D), F32)
        ops.vit_tokens(pe, self.p("vision_model/embeddings/class_embedding"),
                       self.p("vision_model/embeddings/position_embedding/embedding"), tok, B, N, D)
        x = A.alloc((m, D), F32)
        ops.layernorm_f32(tok, self.p("vision_model/pre_layrnorm/scale"), self.p("vision_model/pre_layrnorm/bias"), x, m, D,
                          eps=cfg.layer_norm_eps)
        for t in (patches, pe, tok):
            A.release(t)
        for i in range(cfg.num_hidden_layers):
            b = f"vision_model/encoder/layers/{i}"
            ln = A.alloc((m, D), BF16)
            ops.layernorm_fwd(x, self.p(b + "/layer_norm1/scale"), self.p(b + "/layer_norm1/bias"), ln, m, D)
            qkv = A.alloc((m, 3 * D), BF16)
            ops.igemm(a0=ln, wt=self.w[b + "/self_attn/qkv"], n=3 * D, c0=D, m=m, bias=self.qkv_bias[b + "/self_attn/qkv"],
                      out_bf16=qkv)
            ao = A.alloc((m, D), BF16)
            ops.attention_fwd(qkv, qkv[:, D:], qkv[:, 2 * D:], ao, B, H, L, L, 3 * D, 3 * D, 3 * D, D, causal=False)
            h1 = A.alloc((m, D), F32)
            ops.igemm(a0=ao, wt=self.w[b + "/self_attn/out_proj"], n=D, c0=D, m=m,
                      bias=self.p(b + "/self_attn/out_proj/bias"), residual=x, out_f32=h1)
            ops.layernorm_fwd(h1, self.p(b + "/layer_norm2/scale"), self.p(b + "/layer_norm2/bias"), ln, m, D)
            f1 = A.alloc((m, I), F32)
            ops.igemm(a0=ln, wt=self.w[b + "/mlp/fc1"], n=I, c0=D, m=m, bias=self.p(b + "/mlp/fc1/bias"), out_f32=f1)
            fa = A.alloc((m, I), BF16)
            ops.act_bf16(f1, fa, cfg.hidden_act)
            x2 = A.alloc((m, D), F32)
            ops.igemm(a0=fa, wt=self.w[b + "/mlp/fc2"], n=D, c0=I, m=m, bias=self.p(b + "/mlp/fc2/bias"), residual=h1,
                      out_f32=x2)
            for t in (ln, qkv, ao, h1, f1, fa, x):
                A.release(t)
            x = x2
        cls = A.alloc((B, D), F32)
        ops.gather_rows(x, torch.arange(B, device=self.device, dtype=torch.int64) * L, cls)       # the CLS token rows
        cls_ln = A.alloc((B, D), BF16)
        ops.layernorm_fwd(cls, self.p("vision_model/post_layernorm/scale"), self.p("vision_model/post_layernorm/bias"),
                          cls_ln, B, D)
        feats = torch.empty(B, cfg.projection_dim, dtype=F32, device=self.device)
        ops.igemm(a0=cls_ln, wt=self.w["proj"], n=cfg.projection_dim, c0=D, m=B, out_f32=feats)
        for t in (x, cls, cls_ln):
            A.release(t)
        return feats

    def features(self, images_u8, transform: int = IDENTITY, chunk: int = 32) -> torch.Tensor:
        """uint8 NHWC device batch -> ``get_image_features`` of ``transform(image)`` preprocessed on the device"""
        return torch.cat([self.image_features(preprocess_device(images_u8[s:s + chunk], self.cfg.image_size, transform))
                          for s in range(0, len(images_u8), chunk)])


def _maybe_load_laion(cfg, flat, cache):
    """Reference ``laion.load_weights`` / ``set_weights`` (:21-52) when the weight file is present (never downloaded)."""
    path = os.path.join(cache, "sac+logos+ava1-l14-linearMSE.pth")
    if cfg.projection_dim != 768 or not os.path.exists(path):
        return
    table, _ = param_offsets(cfg)
    weights = torch.load(path, map_location="cpu")
    for i, layer in enumerate((0, 2, 4, 6, 7)):
        for leaf, t in (("kernel", weights[f"layers.{layer}.weight"].t()), ("bias", weights[f"layers.{layer}.bias"])):
            off, shape = table[f"aesthetic/Dense_{i}/{leaf}"]
            flat[off:off + int(np.prod(shape))] = t.contiguous().reshape(-1).float()


class AestheticScorer(CLIPImageTower):
    """the image tower followed by L2 normalisation and the LAION ``AestheticClassifier``"""
    HEAD = True

    def __init__(self, cfg: CLIPVisionConfig = VIT_L14, flat_params: torch.Tensor = None, device="cuda", seed: int = 0,
                 cache: str = "cache"):
        if flat_params is None:
            flat_params = init_flat_params(cfg, seed)
            _maybe_load_laion(cfg, flat_params, cache)
        super().__init__(cfg, flat_params, device, seed)

    @torch.no_grad()
    def score_features(self, feats: torch.Tensor) -> torch.Tensor:
        """image features -> L2 normalise -> AestheticClassifier -> [B, 1]"""
        A = self.arena
        B, k = feats.shape
        cur = A.alloc((B, k), F32)
        ops.l2norm_rows(feats, cur)
        for i, n in enumerate(HEAD_SIZES):
            nxt = A.alloc((B, n), F32)
            ops.dense_small(cur, self.p(f"aesthetic/Dense_{i}/kernel"), self.p(f"aesthetic/Dense_{i}/bias"), nxt, B, k, n)
            A.release(cur)
            cur, k = nxt, n
        out = cur.clone()
        A.release(cur)
        return out

    def __call__(self, images, chunk: int = 32):
        """float images [N, H, W, 3] in [0, 1] (or uint8) -> scores float32 numpy [N, 1] (reference ``_wrapper`` :86-91)"""
        u8 = torch.from_numpy(to_uint8(images)).to(self.device)
        # a CPU tower exists only in host dry runs on emulated ops, where the host preprocess is the reference
        prep = preprocess_device if self.device.type == "cuda" else \
            (lambda x, size: torch.from_numpy(preprocess(x.numpy(), size)))
        return np.concatenate([self.score_features(self.image_features(
            prep(u8[s:s + chunk], self.cfg.image_size))).cpu().numpy() for s in range(0, len(u8), chunk)])


class CLIPConsistency:
    """``FlaxCLIPModel(**processor(text=prompts, images=images, padding=True)).logits_per_image.diagonal()`` (3P
    transformers==4.28.1, reference ``callbacks.py:122-140``) on the kernels: the image tower's features and the text
    tower's hidden state at the first position of the largest token id (transformers' ``argmax`` pooling; the tokenizer's
    end-of-text id 49407 is its largest), each projected without bias, ``exp(logit_scale) cos(image, text)``.  Prompts
    are tokenised to 77 positions: causal attention makes every position up to the end-of-text token independent of the
    padding after it, so this equals the reference's ``padding=True``; a longer prompt raises."""
    MAX_TOKENS = 77
    LOGIT_SCALE_INIT = 2.6592

    def __init__(self, vision_cfg: CLIPVisionConfig = VIT_B32, text_cfg=None, device="cuda", seed: int = 0,
                 tokenizer=None):
        from .text_encoder import CLIP_B32_TEXT, CLIPTextEncoder
        from .utils.text_stub import StubTokenizer
        text_cfg = text_cfg or CLIP_B32_TEXT
        assert text_cfg.max_position_embeddings >= self.MAX_TOKENS
        self.device = torch.device(device)
        self.vision = CLIPImageTower(vision_cfg, device=self.device, seed=seed)
        self.text = CLIPTextEncoder(text_cfg, device=self.device, seed=seed)
        self.tokenizer = tokenizer or StubTokenizer()
        D, P = text_cfg.hidden_size, vision_cfg.projection_dim
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.text_projection = (torch.randn(D, P, generator=g) / np.sqrt(D)).to(self.device)   # Flax [in, out]
        self.logit_scale = float(np.float32(self.LOGIT_SCALE_INIT))

    def token_ids(self, prompts):
        """[B, 77] ids and the pooled position of each row; a prompt whose end-of-text token falls past 77 raises"""
        ids = np.asarray(self.tokenizer(list(prompts), padding="max_length", max_length=self.MAX_TOKENS + 1,
                                        truncation=True, return_tensors="np").input_ids)
        pos = ids.argmax(-1)
        if (pos >= self.MAX_TOKENS).any():
            raise ValueError(f"prompt {list(prompts)[int(np.argmax(pos))]!r} is longer than {self.MAX_TOKENS} tokens")
        return ids[:, :self.MAX_TOKENS], pos

    @torch.no_grad()
    def text_features(self, prompts) -> torch.Tensor:
        ids, pos = self.token_ids(prompts)
        B, L = ids.shape
        D, P = self.text.cfg.hidden_size, self.vision.cfg.projection_dim
        hidden = self.text.encode(ids).reshape(B * L, D)
        pooled = torch.empty(B, D, dtype=F32, device=self.device)
        ops.gather_rows(hidden, torch.from_numpy(np.arange(B) * L + pos).to(self.device, torch.int64), pooled)
        out = torch.empty(B, P, dtype=F32, device=self.device)
        ops.dense_small(pooled, self.text_projection, None, out, B, D, P)
        return out

    @torch.no_grad()
    def __call__(self, images_u8: torch.Tensor, prompts) -> np.ndarray:
        """uint8 NHWC device batch and one prompt per image -> float32 [N] logits"""
        assert len(prompts) == len(images_u8)
        img = self.vision.features(images_u8)
        out = torch.empty(len(images_u8), dtype=F32, device=self.device)
        ops.scaled_cosine(img, self.text_features(prompts), self.logit_scale, out)
        return out.cpu().numpy()
