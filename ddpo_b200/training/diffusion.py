"""Reward-weighted-regression (RWR) update of the denoiser -- drop-in mirror of the reference's
``ddpo/training/diffusion.py`` (``train_step`` :6-102, ``vae_decode`` :105-112, ``text_encode`` :115-116) and of the
``TrainState`` / optimizer chain ``pipeline/finetune.py:88-110`` builds (3P flax ``TrainState`` +
``optax.chain(clip_by_global_norm, adamw(mu_dtype=bf16))``).

Same call shape::

    state, loss, train_rng = train_step(state, text_encoder_params, batch, train_rng, noise_scheduler_state,
                                        (noise_scheduler, text_encoder, train_cfg, guidance_scale), weights=None)

``batch["vae"]`` holds the stored posterior moments ``[B, h, w, 8]`` (mean | logvar, channels-last, as the reference's
bucket datasets store them); the text side is either ``batch["input_ids"]`` / ``batch["uncond_text"]`` run through the
``text_encoder`` callable exactly as the reference does (:47-51, :64-68), or -- when the caller has embedded the
prompts already -- ``batch["prompt_embeds"]`` / ``batch["uncond_embeds"]``.

GPU design: posterior sample, noise and ``add_noise`` are ONE kernel (jax-compatible threefry in registers); the
conditional and unconditional U-Net applications run as one batch of 2B with context ``[uncond ; cond]``; the MSE on the
CFG-combined prediction and its gradient are one kernel; forward + loss + backward replay as one CUDA graph; the
``lax.pmean(grad)`` (:96) is one NCCL all-reduce of the flat gradient folded into the fused clip+AdamW kernel.
"""
from typing import Any, Dict

import numpy as np
import torch

from .. import ops
from ..ops import graph_step   # host-side control: stays the real one where ``ops`` is swapped for an emulator
from . import distributed
from .policy_gradient import AccumulatingTrainState, AdamWConfig  # noqa: F401  (same optimizer chain)
from ..unet import UNet


class TrainState(AccumulatingTrainState):
    """``flax.training.train_state.TrainState`` as ``pipeline/finetune.py:104-108`` creates it: every
    ``apply_gradients`` is an optimizer update (no accumulation)."""

    def apply_gradients(self, *, grads=None, **kwargs):
        return super().apply_gradients(grads=grads, do_update=True, n_micro=1)


class _StepGraph:
    def __init__(self, unet: UNet, b, h, w, ctx_len, ctx_dim, train_cfg, weighted):
        dev = unet.device
        self.nb = 2 * b if train_cfg else b
        self.moments = torch.empty(b, h, w, 8, device=dev)
        self.ts = torch.empty(b, dtype=torch.int32, device=dev)
        self.keys = torch.zeros(2, 2, dtype=torch.int32, device=dev)       # [sample_rng ; noise_rng]
        self.ctx = torch.empty(self.nb, ctx_len, ctx_dim, device=dev)
        self.noise = torch.empty(b, 4, h, w, device=dev)
        self.noisy = torch.empty(b, 4, h, w, device=dev)
        self.lat_in = torch.empty(self.nb, 4, h, w, device=dev)
        self.ts_in = torch.empty(self.nb, dtype=torch.int32, device=dev)
        self.eps = torch.empty(self.nb, 4, h, w, device=dev)
        self.d_eps = torch.zeros(self.nb, 4, h, w, device=dev)
        self.weights = torch.empty(b, device=dev) if weighted else None
        self.loss = torch.zeros(1, device=dev)
        self.per_sample = torch.zeros(b, device=dev)
        self.ws = ops.rwr_workspace(b, dev)
        self.graph = None   # what ops.graph_step returned


_GRAPHS: Dict[Any, _StepGraph] = {}
USE_CUDA_GRAPH = True
VAE_SCALING = 0.18215  # reference :20


def _run_body(unet: UNet, G: _StepGraph, b, train_cfg, alphas_cumprod, guidance_scale):
    n = G.noise[0].numel()
    ops.rwr_noisy_latents(G.moments, G.keys[0], G.keys[1], G.ts, alphas_cumprod, G.noise, G.noisy, scaling=VAE_SCALING)
    if train_cfg:
        G.lat_in[:b].copy_(G.noisy)
        G.lat_in[b:].copy_(G.noisy)
        G.ts_in[:b].copy_(G.ts)
        G.ts_in[b:].copy_(G.ts)
    else:
        G.lat_in.copy_(G.noisy)
        G.ts_in.copy_(G.ts)
    unet.prepare_context(G.ctx)
    tape = []
    unet.forward(G.lat_in, G.ts_in, out=G.eps, tape=tape)
    eps, d_eps = G.eps.view(G.nb, n), G.d_eps.view(G.nb, n)
    noise = G.noise.view(b, n)
    if train_cfg:
        ops.rwr_mse_loss(eps[:b], eps[b:], noise, float(guidance_scale), G.loss, G.ws, weights=G.weights,
                         per_sample=G.per_sample, d_eps_u=d_eps[:b], d_eps_c=d_eps[b:])
    else:  # noise_pred = cond output (:81): eps_u slot with guidance 0 reproduces it exactly
        ops.rwr_mse_loss(eps, eps, noise, 0.0, G.loss, G.ws, weights=G.weights, per_sample=G.per_sample,
                         d_eps_u=d_eps, d_eps_c=None)
    unet.backward(tape, G.d_eps)


def _encode(text_encoder, text_encoder_params, ids):
    out = text_encoder(ids, params=text_encoder_params, train=False)
    return out[0] if isinstance(out, (tuple, list)) else out


def train_step(state: AccumulatingTrainState, text_encoder_params, batch, train_rng, noise_scheduler_state,
               static_broadcasted, weights=None):
    noise_scheduler, text_encoder, train_cfg, guidance_scale = static_broadcasted
    unet = state.apply_fn
    dev = unet.device
    # ---- key lineage (:14, :23): dropout_rng is unused (dropout 0), sample_rng feeds the posterior AND is split again
    train_rng = tuple(int(v) for v in np.asarray(train_rng).reshape(-1)[:2])
    _dropout_rng, sample_rng, new_train_rng = ops.threefry_split(train_rng, 3)
    noise_rng, timestep_rng = ops.threefry_split(sample_rng, 2)
    moments = batch["vae"]
    moments = moments if torch.is_tensor(moments) else torch.as_tensor(np.asarray(moments, np.float32))
    b, h, w, c2 = moments.shape
    assert c2 == 8, "batch['vae'] must be [B, h, w, 8] posterior moments (mean | logvar, channels last)"
    timesteps = ops.threefry_randint(timestep_rng, b, 0, noise_scheduler.config.num_train_timesteps)  # :27-32
    if "prompt_embeds" in batch:
        emb = batch["prompt_embeds"]
        unc = batch.get("uncond_embeds") if train_cfg else None
    else:
        emb = _encode(text_encoder, text_encoder_params, batch["input_ids"])                  # :45-51
        unc = _encode(text_encoder, text_encoder_params, batch["uncond_text"]) if train_cfg else None  # :62-68
    emb = torch.as_tensor(emb)
    if train_cfg:
        assert unc is not None, "train_cfg needs batch['uncond_text'] or batch['uncond_embeds']"
        unc = torch.as_tensor(unc)
    weighted = weights is not None
    key = (id(unet), b, h, w, tuple(emb.shape[1:]), bool(train_cfg), weighted)
    G = _GRAPHS.get(key)
    if G is None:
        G = _GRAPHS[key] = _StepGraph(unet, b, h, w, emb.shape[1], emb.shape[2], bool(train_cfg), weighted)
    G.moments.copy_(moments.to(dev, torch.float32), non_blocking=True)
    G.ts.copy_(torch.tensor(timesteps, dtype=torch.int32), non_blocking=True)
    G.keys.copy_(ops.key_tensor([sample_rng, noise_rng], "cpu"), non_blocking=True)
    if train_cfg:
        G.ctx[:b].copy_(unc.to(dev, torch.float32))
        G.ctx[b:].copy_(emb.to(dev, torch.float32))
    else:
        G.ctx.copy_(emb.to(dev, torch.float32))
    if weighted:
        wt = torch.as_tensor(np.asarray(weights, np.float32) if not torch.is_tensor(weights) else weights)
        assert wt.numel() == b, "loss.size == weights.size (:88)"
        G.weights.copy_(wt.reshape(b).to(dev, torch.float32))
    ac = noise_scheduler_state.common.alphas_cumprod
    sig = (float(guidance_scale), id(ac))

    def body():
        _run_body(unet, G, b, bool(train_cfg), ac, guidance_scale)

    G.graph = graph_step(G.graph, sig, body, USE_CUDA_GRAPH, protect=state.grad_acc)
    loss = G.loss.clone()
    distributed.pmean_(loss)                                   # :95
    if isinstance(state, TrainState):
        state.apply_gradients(grads=None)                      # :98 (pmean of the gradient happens inside)
    else:
        state.apply_gradients(grads=None, do_update=True, n_micro=1)
    train_step.last = {"timesteps": timesteps, "noise": G.noise, "noisy_latents": G.noisy, "per_sample": G.per_sample}
    return state, loss[0], new_train_rng


def vae_decode(latents, vae_params, apply_fn, decode_fn=None):
    """Reference :105-112.  ``apply_fn`` is the B200 VAE decoder object (``ddpo_b200.vae.VAEDecoder``) or any callable
    ``(latents NCHW) -> images NHWC in [0,1]``; ``vae_params`` / ``decode_fn`` are accepted for signature parity."""
    fn = getattr(apply_fn, "decode_to_images", apply_fn)
    return fn(latents)


def text_encode(input_ids, params, text_encoder):
    """Reference :115-116."""
    out = text_encoder(input_ids, params=params)
    return out[0] if isinstance(out, (tuple, list)) else out


def patch_scheduler(pipeline):
    """Reference :119-132: swap the pipeline's scheduler for the log-prob DDIM scheduler with the same config."""
    from ..diffusers_patch import DDIMScheduler
    c = pipeline.scheduler.config
    pipeline.scheduler = DDIMScheduler(num_train_timesteps=c.num_train_timesteps, beta_start=c.beta_start,
                                       beta_end=c.beta_end, beta_schedule=c.beta_schedule,
                                       trained_betas=c.trained_betas, set_alpha_to_one=c.set_alpha_to_one,
                                       steps_offset=c.steps_offset, prediction_type=c.prediction_type,
                                       device=getattr(pipeline.scheduler, "device", "cuda"))
