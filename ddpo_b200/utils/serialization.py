"""Model construction and U-Net checkpoints -- the subset of the reference's ``ddpo/utils/serialization.py`` the hot
path's drivers call: ``load_unet`` (:320-371), ``load_finetuned_stable_diffusion`` (:247-273), ``save_unet``
(:276-297), ``get_latest_epoch`` / ``load_flax_model`` (:300-317), and the Flax checkpoint written by
``pipeline/policy_gradient.py:457-464`` (3P ``flax.training.checkpoints.save_checkpoint_multiprocess`` ->
``checkpoints/checkpoint_<step>``, a msgpack of the nested parameter dict).

There is no network in this build: ``load_unet`` ingests a LOCAL diffusers checkpoint directory when ``pretrained_model``
resolves to one (``utils/pretrained.py``: Flax msgpack or PyTorch safetensors), creates RANDOM-INIT weights only on the
explicit ``random:<architecture>`` opt-in (the benchmark's stated synthetic setting), and restores U-Nets this package saved.
On-disk formats follow the reference: ``unet_<epoch>.pkl`` is a pickle of the nested ``{module: {...: ndarray}}`` dict
(Flax names, ``kernel`` = ``[in, out]`` / HWIO), ``checkpoint_<step>`` is flax==0.6.9's ``msgpack_serialize`` layout
(ndarray = ExtType 1 holding ``packb((shape, dtype.name, bytes))``) -- both loadable by the reference's own readers.
"""
import os
import pickle
from collections import namedtuple

import numpy as np
import torch

from .. import unet_spec
from . import filesystem
from .timer import Timer

StableModels = namedtuple("StableModels", "tokenizer text_encoder vae unet")
StableParams = namedtuple("StableParams", "vae_params unet_params")

MODEL_CONFIGS = {
    "stabilityai/stable-diffusion-2-base": "SD2_BASE",
    "flax/stable-diffusion-2-1": "SD2_BASE",
    # SD1.x: 8 heads at every level (head dims 40, 80, 160), 768-wide CLIP-L context; the reference's default model
    "duongna/stable-diffusion-v1-4-flax": "SD1",
    "CompVis/stable-diffusion-v1-4": "SD1",
    "runwayml/stable-diffusion-v1-5": "SD1",
    "tiny": "TINY",
    "small": "SMALL",
}


def unet_config_for(pretrained_model):
    name = MODEL_CONFIGS.get(pretrained_model)
    if name is None:
        raise ValueError(f"[ utils/serialization ] no U-Net architecture registered for {pretrained_model!r}; known: "
                         f"{sorted(MODEL_CONFIGS)}")
    return getattr(unet_spec, name)


# ------------------------------------------------------------------ param trees ----
def params_tree(flat, cfg):
    """flat fp32 buffer -> nested dict of numpy arrays keyed by the Flax module path."""
    flat = flat.detach().cpu() if torch.is_tensor(flat) else torch.as_tensor(flat)
    tree = {}
    for name, v in unet_spec.views(flat, cfg).items():
        node = tree
        parts = name.split("/")
        for p in parts[:-1]:
            node = node.setdefault(p, {})
        node[parts[-1]] = v.numpy().copy()
    return tree


def flat_from_tree(tree, cfg):
    table, total = unet_spec.param_offsets(cfg)
    flat = torch.zeros(total, dtype=torch.float32)
    for name, (off, shape) in table.items():
        node = tree
        for p in name.split("/"):
            node = node[p]
        arr = np.asarray(node, np.float32)
        assert tuple(arr.shape) == tuple(shape), f"{name}: checkpoint shape {arr.shape} != {shape}"
        flat[off:off + arr.size] = torch.from_numpy(arr.reshape(-1))
    return flat


def n_params(tree):
    """``utils.n_params`` (reference ``ddpo/utils/array.py:18-19``)."""
    if isinstance(tree, dict):
        return sum(n_params(v) for v in tree.values())
    return int(np.asarray(tree).size)


# ------------------------------------------------------------- flax msgpack I/O ----
def _pack_default(x):
    import msgpack
    if isinstance(x, np.ndarray):
        return msgpack.ExtType(1, msgpack.packb((list(x.shape), x.dtype.name, x.tobytes("C")), use_bin_type=True))
    if isinstance(x, np.generic):
        return msgpack.ExtType(3, msgpack.packb((x.dtype.name, x.tobytes()), use_bin_type=True))
    raise TypeError(f"cannot serialise {type(x)}")


def _unpack_ext(code, data):
    import msgpack
    if code == 1:
        shape, dtype, buf = msgpack.unpackb(data, raw=False)
        return np.frombuffer(buf, dtype=np.dtype(dtype)).reshape(shape).copy()
    if code == 3:
        dtype, buf = msgpack.unpackb(data, raw=False)
        return np.frombuffer(buf, dtype=np.dtype(dtype))[0]
    return msgpack.ExtType(code, data)


def msgpack_serialize(tree):
    import msgpack
    return msgpack.packb(tree, default=_pack_default, strict_types=True, use_bin_type=True)


def msgpack_restore(buf):
    import msgpack
    return msgpack.unpackb(buf, ext_hook=_unpack_ext, raw=False, strict_map_key=False)


def save_checkpoint(ckpt_dir, target, step, prefix="checkpoint_", keep=1, overwrite=False):
    """``flax.training.checkpoints.save_checkpoint`` semantics for a parameter tree (atomic rename, ``keep`` newest)."""
    ckpt_dir = filesystem.localize(ckpt_dir)
    os.makedirs(ckpt_dir, exist_ok=True)
    path = os.path.join(ckpt_dir, f"{prefix}{step}")
    if os.path.exists(path) and not overwrite:
        raise FileExistsError(f"checkpoint {path} exists and overwrite=False")
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        f.write(msgpack_serialize(target))
    os.replace(tmp, path)
    steps = sorted(int(f[len(prefix):]) for f in os.listdir(ckpt_dir)
                   if f.startswith(prefix) and f[len(prefix):].isdigit())
    for s in steps[: max(0, len(steps) - int(min(keep, 1e9)))]:
        os.remove(os.path.join(ckpt_dir, f"{prefix}{s}"))
    return path


def save_checkpoint_multiprocess(ckpt_dir, target, step, prefix="checkpoint_", keep=1, overwrite=False):
    """Only process 0 writes (3P flax ``save_checkpoint_multiprocess``); the others wait at a barrier."""
    from ..training import distributed
    path = None
    if distributed.rank() == 0:
        path = save_checkpoint(ckpt_dir, target, step, prefix, keep, overwrite)
    if distributed.is_distributed():
        torch.distributed.barrier()
    return path


def restore_checkpoint(ckpt_dir, step=None, prefix="checkpoint_"):
    ckpt_dir = filesystem.localize(ckpt_dir)
    if step is None:
        steps = [int(f[len(prefix):]) for f in os.listdir(ckpt_dir) if f.startswith(prefix) and f[len(prefix):].isdigit()]
        if not steps:
            raise FileNotFoundError(f"no checkpoints under {ckpt_dir}")
        step = max(steps)
    with open(os.path.join(ckpt_dir, f"{prefix}{step}"), "rb") as f:
        return msgpack_restore(f.read())


# ------------------------------------------------------------------ unet_*.pkl ----
def save_unet(savepath, unet_params, epoch=0, all_workers=False, cache="logs"):
    """Reference :276-297.  ``unet_params`` is the nested dict (``params_tree``)."""
    from ..training import distributed
    local_path = filesystem.localize(savepath, cache)
    os.makedirs(local_path, exist_ok=True)
    fullpath = os.path.join(local_path, f"unet_{epoch}.pkl")
    print(f"[ utils/serialization ] Saving unet to {fullpath}")
    if distributed.rank() == 0 or all_workers:
        with open(fullpath, "wb") as f:
            pickle.dump(unet_params, f)
        return local_path, None
    return None, None


def get_latest_epoch(loadpath):
    loadpath, prefix = os.path.split(loadpath)
    fnames = [f for f in filesystem.ls(loadpath) if prefix in f]
    return max(int(f.split("_")[-1].split(".pkl")[0]) for f in fnames)


def load_flax_model(loadpath, epoch="latest"):
    timer = Timer()
    if epoch == "latest":
        epoch = get_latest_epoch(loadpath)
        print(f"[ utils/serialization ] Found latest epoch: {epoch}")
    fullpath = loadpath + f"_{epoch}.pkl"
    print(f"[ utils/serialization ] Loading model from {fullpath}")
    params = filesystem.unpickle(fullpath)
    print(f"[ utils/serialization ] Done | {timer():.3f} seconds")
    return params


# --------------------------------------------------------------------- loaders ----
RANDOM_PREFIX = "random:"
ALLOW_RANDOM_ENV = "DDPO_ALLOW_RANDOM_INIT"


def load_unet(loadpath, epoch="latest", pretrained_model="stabilityai/stable-diffusion-2-base", dtype="float32",
              cache="cache", device="cuda", seed=0, with_vae=True, text_encoder="clip"):
    """Reference :320-371: returns ``(pipeline, params)`` with ``params`` = ``{"unet", "vae", "text_encoder",
    "scheduler"}``.

    Weights: ``pretrained_model`` is resolved to a LOCAL diffusers checkpoint directory (a path, ``<cache>/<id>`` or the
    hub cache layout under ``cache`` -- there is no network to download from); its U-Net / VAE decoder / text encoder /
    scheduler config / tokenizer are ingested by ``utils/pretrained.py`` (Flax msgpack or PyTorch safetensors / .bin).
    Random initialisation is an explicit opt-in: ``pretrained_model="random:<architecture>"`` (e.g.
    ``random:stabilityai/stable-diffusion-2-base``), the test-sized ``"tiny"`` / ``"small"``, or
    ``$DDPO_ALLOW_RANDOM_INIT=1``; anything else without a checkpoint on disk raises.  ``loadpath`` then overlays a
    saved ``unet_<epoch>.pkl`` as in the reference."""
    from ..diffusers_patch import DDIMScheduler, StableDiffusionPipeline
    from ..unet import UNet
    from . import pretrained
    from .text_stub import StubTextEncoder, StubTokenizer
    ckpt_dir = pretrained.resolve_dir(pretrained_model, cache)
    sched_kw = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                    set_alpha_to_one=False, steps_offset=1, prediction_type="epsilon")
    vae_flat = vae_enc_flat = vae_cfg = text_flat = text_cfg = tokenizer = None
    if ckpt_dir is not None:
        print(f"[ utils/serialization ] Loading {pretrained_model} from {ckpt_dir} | dtype: {dtype}")
        cfg, flat = pretrained.load_unet_weights(ckpt_dir)
        sched_kw.update(pretrained.load_scheduler_config(ckpt_dir))
        if with_vae and os.path.isdir(os.path.join(ckpt_dir, "vae")):
            vae_cfg, vae_flat = pretrained.load_vae_decoder_weights(ckpt_dir)
            try:
                _, vae_enc_flat = pretrained.load_vae_decoder_weights(ckpt_dir, part="encoder")
            except KeyError:      # a decoder-only checkpoint: the encoder stays random-init
                vae_enc_flat = None
        if text_encoder == "clip" and os.path.isdir(os.path.join(ckpt_dir, "text_encoder")):
            text_cfg, text_flat = pretrained.load_text_encoder_weights(ckpt_dir)
        tokenizer = pretrained.load_tokenizer(ckpt_dir)
        arch = pretrained_model
    else:
        explicit = str(pretrained_model).startswith(RANDOM_PREFIX)
        arch = str(pretrained_model)[len(RANDOM_PREFIX):] if explicit else pretrained_model
        if not (explicit or arch in ("tiny", "small") or os.environ.get(ALLOW_RANDOM_ENV) == "1"):
            raise FileNotFoundError(
                f"[ utils/serialization ] no local checkpoint for {pretrained_model!r} (looked for <dir>/unet/config.json at "
                f"the path itself and under {cache!r}); there is no network to download it.  For random-init weights of "
                f"that architecture say pretrained_model='{RANDOM_PREFIX}{pretrained_model}' or set {ALLOW_RANDOM_ENV}=1.")
        cfg = unet_config_for(arch)
        print(f"[ utils/serialization ] Building {arch} ({unet_spec.num_params(cfg) / 1e6:.1f}M-parameter U-Net) with "
              f"RANDOM-INIT weights | dtype: {dtype}")
        flat = unet_spec.init_flat_params(cfg, seed)
    if loadpath:
        tree = load_flax_model(os.path.join(filesystem.localize(loadpath), "unet"), epoch=epoch)
        flat = flat_from_tree(tree, cfg)
    unet = UNet(cfg, flat, device)
    scheduler = DDIMScheduler(device=device, **sched_kw)
    vae = vae_encoder = None
    if with_vae:
        from ..vae import VAEDecoder, VAEEncoder, vae_config_for
        vae = (VAEDecoder(vae_cfg, vae_flat, device=device) if vae_flat is not None
               else VAEDecoder(vae_config_for(arch), device=device, seed=seed + 1))
        if str(device) != "cpu":   # the RWR sampler's "vae" field; the CPU dry runs of the drivers never encode
            vae_encoder = (VAEEncoder(vae_cfg, vae_enc_flat, device=device) if vae_enc_flat is not None
                           else VAEEncoder(vae.cfg, device=device, seed=seed + 3))
    if text_encoder == "clip":
        # the CLIP text tower on the GPU; without tokenizer files the stub tokenizer's ids are folded into its vocabulary
        from ..text_encoder import CLIPTextEncoder, text_config_for
        tenc = (CLIPTextEncoder(text_cfg, text_flat, device=device) if text_flat is not None
                else CLIPTextEncoder(text_config_for(arch), device=device, seed=seed + 2))
    else:
        tenc = StubTextEncoder(cfg.cross_attention_dim)
    pipeline = StableDiffusionPipeline(unet, scheduler, tokenizer=tokenizer or StubTokenizer(), text_encoder=tenc, vae=vae,
                                       vae_scale_factor=8)
    pipeline.vae_encoder = vae_encoder
    params = {"unet": unet.params, "vae": None if vae is None else vae.params,
              "text_encoder": getattr(tenc, "params", {}), "scheduler": scheduler.create_state()}
    return pipeline, params


def load_finetuned_stable_diffusion(name, epoch="latest", pretrained_model="stabilityai/stable-diffusion-2-base",
                                    dtype="float32", cache="cache", device="cuda", seed=0):
    """Reference :247-273: ``((tokenizer, text_encoder, vae, unet), (vae_params, unet_params))``."""
    pipeline, params = load_unet(name, epoch=epoch, pretrained_model=pretrained_model, dtype=dtype, cache=cache,
                                 device=device, seed=seed)
    models = StableModels(pipeline.tokenizer, pipeline.text_encoder, pipeline.vae, pipeline.unet)
    return models, StableParams(params["vae"], params["unet"])
