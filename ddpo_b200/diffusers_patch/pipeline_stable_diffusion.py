"""Trajectory sampler -- drop-in mirror of the reference's patched Stable-Diffusion pipeline
(``ddpo/diffusers_patch/pipeline_flax_stable_diffusion.py``: ``__call__`` :272-367, ``_generate``
:163-270, ``_p_generate`` :372-401): takes prompt *embeddings*, runs T DDIM steps with
classifier-free guidance and returns the whole trajectory plus per-step log-probs

    (final_latents [B,4,h,w], latents [B,T,4,h,w], next_latents [B,T,4,h,w], log_probs [B,T], ts [B,T])

GPU design instead of ``pmap(lax.scan)``: one process per GPU owns its shard of the batch; one
denoising step (U-Net on the 2B CFG batch + fused CFG/DDIM/log-prob/threefry kernel) is captured in
a CUDA graph and replayed T times; the trajectory stays in HBM ([T+1, B, n] buffer, ``latents`` and
``next_latents`` are views of it).  Noise is bit-compatible with ``jax.random`` (same key lineage:
``split`` -> ``normal`` per step, reference :196-197, :232, :252).
"""
from typing import Optional

import numpy as np
import torch

from .. import ops
from ..ops import graph_step   # host-side control: stays the real one where ``ops`` is swapped for an emulator
from ..unet import UNet
from .scheduling_ddim import DDIMScheduler


class StableDiffusionPipeline:
    def __init__(self, unet: UNet, scheduler: DDIMScheduler, tokenizer=None, text_encoder=None, vae=None,
                 vae_scale_factor: int = 8, use_cuda_graph: bool = True):
        self.unet = unet
        self.scheduler = scheduler
        self.tokenizer = tokenizer
        self.text_encoder = text_encoder
        self.vae = vae
        self.vae_scale_factor = vae_scale_factor
        self.safety_checker = None
        self.use_cuda_graph = use_cuda_graph
        self._graphs = {}

    # reference :148-161
    def prepare_inputs(self, prompt):
        if not isinstance(prompt, (str, list)):
            raise ValueError(f"`prompt` has to be of type `str` or `list` but is {type(prompt)}")
        if self.tokenizer is None:
            raise RuntimeError("no tokenizer attached to the pipeline")
        return self.tokenizer(prompt, padding="max_length", max_length=self.tokenizer.model_max_length,
                              truncation=True, return_tensors="np").input_ids

    # ------------------------------------------------------------------ one step ----
    def _step_buffers(self, b, h, w, dev):
        key = (b, h, w)
        if key not in self._graphs:
            n = 4 * h * w
            self._graphs[key] = dict(
                lat_in=torch.empty(2 * b, 4, h, w, device=dev), x_cur=torch.empty(b, n, device=dev),
                x_next=torch.empty(b, n, device=dev), logp=torch.empty(b, device=dev),
                eps=torch.empty(2 * b, 4, h, w, device=dev), t_dev=torch.zeros(1, dtype=torch.int32, device=dev),
                key_dev=torch.zeros(2, dtype=torch.int32, device=dev), ws=ops.ddim_workspace(b, dev), graph=None)
        return self._graphs[key]

    def _one_step(self, S, b, state, ratio, guidance_scale, eta):
        n = S["x_cur"].shape[1]
        S["lat_in"][:b].view(b, n).copy_(S["x_cur"])
        S["lat_in"][b:].view(b, n).copy_(S["x_cur"])
        self.unet.forward(S["lat_in"], S["t_dev"], out=S["eps"])
        eps = S["eps"].view(2 * b, n)
        # context order is [uncond ; cond] (reference :187, :226)
        ops.ddim_step_sample(eps[:b], eps[b:], S["x_cur"], state.common.alphas_cumprod, S["t_dev"],
                             state.final_alpha_cumprod, ratio, guidance_scale, eta, S["key_dev"], S["x_next"],
                             S["logp"], S["ws"], pred=self.scheduler.config.prediction_type)

    # ----------------------------------------------------------------- _generate ----
    @torch.no_grad()
    def _generate(self, prompt_embeds, neg_prompt_embeds, params, rng, num_inference_steps, height, width,
                  guidance_scale, eta, latents=None):
        if height % 8 != 0 or width % 8 != 0:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        dev = self.unet.device
        b = prompt_embeds.shape[0]
        h, w = height // self.vae_scale_factor, width // self.vae_scale_factor
        n = 4 * h * w
        T = int(num_inference_steps)
        sched_state = params["scheduler"] if isinstance(params, dict) and "scheduler" in params else None
        if sched_state is None:
            sched_state = self.scheduler.create_state()
        state = self.scheduler.set_timesteps(sched_state, num_inference_steps=T, shape=(b, 4, h, w))
        ratio = self.scheduler.config.num_train_timesteps // T
        context = torch.cat([neg_prompt_embeds.to(dev, torch.float32), prompt_embeds.to(dev, torch.float32)])
        self.unet.prepare_context(context)
        # ---- key lineage (host threefry; a few dozen 2-word hashes)
        rng = tuple(int(v) for v in rng)
        traj = torch.empty(T + 1, b, n, device=dev)
        if latents is None:
            rng, seed = ops.threefry_split(rng, 2)
            ops.threefry_normal(ops.key_tensor([seed], dev), traj[0].view(-1))
        else:
            if tuple(latents.shape) != (b, 4, h, w):
                raise ValueError(f"Unexpected latents shape, got {tuple(latents.shape)}, expected {(b, 4, h, w)}")
            traj[0].copy_(latents.reshape(b, n))
        if state.init_noise_sigma != 1.0:
            traj[0].mul_(state.init_noise_sigma)
        rng, carry = ops.threefry_split(rng, 2)
        step_keys = []
        for _ in range(T):
            carry, k = ops.threefry_split(carry, 2)
            step_keys.append(k)
        keys_dev = ops.key_tensor(step_keys, dev)
        ts_host = np.asarray(state.timesteps, np.int32)
        ts_dev = torch.as_tensor(ts_host, device=dev)
        logps = torch.empty(T, b, device=dev)

        S = self._step_buffers(b, h, w, dev)
        sig = (float(guidance_scale), float(eta), T, id(state.common.alphas_cumprod), self.scheduler.config.prediction_type)

        def step():
            self._one_step(S, b, state, ratio, float(guidance_scale), float(eta))

        S["x_cur"].copy_(traj[0])
        for s in range(T):
            S["t_dev"].copy_(ts_dev[s:s + 1])
            S["key_dev"].copy_(keys_dev[s])
            S["graph"] = graph_step(S["graph"], sig, step, self.use_cuda_graph)
            traj[s + 1].copy_(S["x_next"])
            logps[s].copy_(S["logp"])
            S["x_cur"].copy_(S["x_next"])

        lat = traj[:-1].view(T, b, 4, h, w).permute(1, 0, 2, 3, 4)
        nxt = traj[1:].view(T, b, 4, h, w).permute(1, 0, 2, 3, 4)
        final = traj[T].view(b, 4, h, w)
        log_probs = logps.permute(1, 0)
        ts = ts_dev.view(1, T).expand(b, T)
        return final, lat, nxt, log_probs, ts

    # ------------------------------------------------------------------ __call__ ----
    def __call__(self, prompt_embeds, neg_prompt_embeds, params, prng_seed, num_inference_steps: int = 50,
                 height: Optional[int] = None, width: Optional[int] = None, guidance_scale=7.5, eta=0.0,
                 latents=None, jit: bool = False):
        height = height or self.unet.cfg.sample_size * self.vae_scale_factor
        width = width or self.unet.cfg.sample_size * self.vae_scale_factor
        # The reference shards inputs over a leading local-device axis for pmap (jit=True).  Here one
        # process drives one GPU, so that axis -- if present -- has size 1 and is carried through.
        sharded = prompt_embeds.dim() == 4
        if sharded:
            assert prompt_embeds.shape[0] == 1, "one process per GPU: the leading device axis must be 1"
            prompt_embeds, neg_prompt_embeds = prompt_embeds[0], neg_prompt_embeds[0]
            prng_seed = np.asarray(prng_seed).reshape(-1, 2)[0]
            if latents is not None:
                latents = latents[0]
        gs = float(np.asarray(guidance_scale).reshape(-1)[0])
        et = float(np.asarray(eta).reshape(-1)[0])
        out = self._generate(prompt_embeds, neg_prompt_embeds, params, prng_seed, num_inference_steps, height, width,
                             gs, et, latents)
        if sharded:
            out = tuple(o.unsqueeze(0) for o in out)
        return out


FlaxStableDiffusionPipeline = StableDiffusionPipeline
