"""PPO update of the denoising policy -- drop-in mirror of the reference's
``ddpo/training/policy_gradient.py`` (``AccumulatingTrainState`` :13-57, ``train_step`` :63-146) and of
the optimizer chain built in ``pipeline/policy_gradient.py:130-150``.

Same call shape::

    state, info = train_step(state, batch, noise_scheduler_state, noise_scheduler, train_cfg,
                             guidance_scale, eta, clip_range, do_opt_update)

``batch`` carries ``latents, next_latents [B,4,h,w]``, ``ts [B]``, ``log_probs, advantages [B]``,
``prompt_embeds, uncond_embeds [B,77,D]`` (``pipeline/policy_gradient.py:415-423``); ``info`` has
``approx_kl, clipfrac, loss``.

GPU design: the conditional and unconditional U-Net applications of ``compute_loss`` (:87-102) run as
ONE batch of 2B with context ``[uncond ; cond]`` -- the very same kernels, tiles and reduction orders as
the sampler, so on an unchanged policy ``ratio == 1`` bit-exactly.  Forward, fused log-prob, PPO loss and
the whole backward are captured in one CUDA graph; weight gradients are accumulated straight into the
flat fp32 ``grad_acc`` buffer by the wgrad epilogues (``grad_acc += g`` costs no extra pass); the data-
parallel ``lax.pmean(grad)`` (:141) becomes ONE NCCL all-reduce of that buffer per optimizer update
(the mean is linear, so reducing the accumulated sum equals reducing every micro-step).
"""
from dataclasses import dataclass
from typing import Any, Dict, Union

import torch

from .. import ops
from ..ops import graph_step   # host-side control: stays the real one where ``ops`` is swapped for an emulator
from . import distributed
from ..unet import UNet

ADV_CLIP_MAX = 10.0  # applied inside the CUDA PPO kernel (reference :60,121)


@dataclass
class AdamWConfig:
    """optax.chain(clip_by_global_norm(max_grad_norm), adamw(..., mu_dtype=bfloat16)) hyper-parameters
    (reference pipeline/policy_gradient.py:130-150; defaults config/base.py:90-95)."""
    learning_rate: float = 1e-5
    b1: float = 0.9
    b2: float = 0.999
    eps: float = 1e-8
    weight_decay: float = 1e-4
    max_grad_norm: float = 1.0


@dataclass
class AdafactorConfig:
    """optax.chain(clip_by_global_norm(max_grad_norm), adafactor(learning_rate, weight_decay_rate=weight_decay))
    hyper-parameters, every other adafactor argument at its optax default (reference pipeline/policy_gradient.py:132-150).
    As in optax, the weight decay is added after the learning-rate scale: each update shrinks p by weight_decay * p."""
    learning_rate: float = 1e-5
    weight_decay: float = 1e-4
    max_grad_norm: float = 1.0
    min_dim_size_to_factor: int = 128


class AccumulatingTrainState:
    """Accumulates gradients over several ``train_step`` calls and applies them when ``do_update``
    (reference :13-57).  ``params`` / ``grad_acc`` are the U-Net's flat fp32 buffers -- or, on a U-Net in LoRA mode
    (``UNet.enable_lora``), its flat adapter buffers, the U-Net itself staying frozen.  ``tx`` picks the optimizer:
    AdamW keeps ``mu`` (bf16) and ``nu`` (fp32) over the whole buffer; Adafactor keeps only its factored second
    moments, one flat fp32 ``state`` laid out by the host planner (``adafactor_leaves`` names its per-tensor views)."""

    def __init__(self, *, step=0, apply_fn: UNet, params=None, tx: Union[AdamWConfig, AdafactorConfig, None] = None,
                 opt_state=None, grad_acc=None, n_acc=0):
        self.step = int(step)
        self.apply_fn = apply_fn
        apply_fn.enable_training()
        lora = apply_fn.lora_rank > 0
        self.params = apply_fn.lora_params if lora else apply_fn.params
        self.tx = tx or AdamWConfig()
        self.grad_acc = apply_fn.lora_grads if lora else apply_fn.grads
        self._table = apply_fn.lora_table if lora else apply_fn.table
        self.n_acc = int(n_acc)
        dev = self.params.device
        if isinstance(self.tx, AdafactorConfig):
            self._plan = ops.adafactor_plan(list(self._table.values()), self.params.numel(),
                                            self.tx.min_dim_size_to_factor)
            self._af_ws = torch.empty(self._plan.workspace_floats, dtype=torch.float32, device=dev)
            if opt_state is None:
                opt_state = {"count": 0, "state": torch.zeros(self._plan.state_floats, dtype=torch.float32, device=dev)}
        elif opt_state is None:
            opt_state = {"count": 0, "mu": torch.zeros(self.params.numel(), dtype=torch.bfloat16, device=dev),
                         "nu": torch.zeros(self.params.numel(), dtype=torch.float32, device=dev)}
        self.opt_state = opt_state
        self._ws = ops.optim_workspace(dev)
        self._sumsq = torch.zeros(1, dtype=torch.float32, device=dev)
        self.last_grad_norm = torch.zeros(1, dtype=torch.float32, device=dev)

    @classmethod
    def create(cls, *, apply_fn, params=None, tx=None, **kw):
        return cls(step=0, apply_fn=apply_fn, params=params, tx=tx, **kw)

    def adafactor_leaves(self):
        """Adafactor only: parameter name -> {"v_row", "v_col"} or {"v"} views of the state, shaped as optax's."""
        views = self._plan.state_views(self.opt_state["state"])
        return dict(zip(self._table, views))

    def apply_gradients(self, *, grads=None, do_update: bool, n_micro: int = 1, **kwargs):
        """``grads`` is accepted for signature parity; the backward pass has already added this step's
        gradient into ``grad_acc`` (fused accumulation), so only the bookkeeping happens here.
        ``n_micro``: how many reference-sized train_step calls the just-finished pass stood for."""
        self.n_acc += int(n_micro)
        if not do_update:
            return self
        world = distributed.allreduce_sum_(self.grad_acc)  # ONE sum over ranks (NCCL over NVLink) per update
        ops.grad_sumsq(self.grad_acc, self._ws, self._sumsq)
        self.opt_state["count"] += 1
        c = self.tx
        if isinstance(c, AdafactorConfig):
            ops.clip_adafactor(self.params, self.grad_acc, self.opt_state["state"], self._plan, self._af_ws, self._sumsq,
                               distributed.grad_scale(self.n_acc, world), c.max_grad_norm, c.learning_rate, c.weight_decay,
                               self.opt_state["count"], norm_out=self.last_grad_norm)
        else:
            ops.clip_adamw(self.params, self.grad_acc, self.opt_state["mu"], self.opt_state["nu"], self._sumsq,
                           distributed.grad_scale(self.n_acc, world), c.max_grad_norm, c.learning_rate, c.b1, c.b2, c.eps,
                           c.weight_decay, self.opt_state["count"], norm_out=self.last_grad_norm)
        self.apply_fn.refresh_weights()
        self.step += 1
        self.n_acc = 0
        return self


class _StepGraph:
    """Static buffers + captured CUDA graph of fwd + log-prob + PPO loss + bwd for one batch shape."""

    def __init__(self, unet: UNet, b, h, w, ctx_len, ctx_dim, train_cfg):
        dev = unet.device
        self.nb = 2 * b if train_cfg else b
        self.lat = torch.empty(b, 4, h, w, device=dev)
        self.nxt = torch.empty(b, 4, h, w, device=dev)
        self.ts = torch.empty(b, dtype=torch.int32, device=dev)
        self.old_logp = torch.empty(b, device=dev)
        self.adv = torch.empty(b, device=dev)
        self.ctx = torch.empty(self.nb, ctx_len, ctx_dim, device=dev)
        self.lat_in = torch.empty(self.nb, 4, h, w, device=dev)
        self.ts_in = torch.empty(self.nb, dtype=torch.int32, device=dev)
        self.eps = torch.empty(self.nb, 4, h, w, device=dev)
        self.d_eps = torch.zeros(self.nb, 4, h, w, device=dev)
        self.logp = torch.empty(b, device=dev)
        self.dlogp = torch.empty(b, device=dev)
        self.info = torch.empty(3, device=dev)
        self.ws = ops.ddim_workspace(b, dev)
        self.graph = None   # what ops.graph_step returned


_GRAPHS: Dict[Any, _StepGraph] = {}
USE_CUDA_GRAPH = True


def _run_body(unet: UNet, G: _StepGraph, b, train_cfg, sched_state, ratio, guidance_scale, eta, clip_range,
              micro_batch=None, pred="epsilon"):
    n = G.lat[0].numel()
    if train_cfg:
        G.lat_in[:b].copy_(G.lat)
        G.lat_in[b:].copy_(G.lat)
        G.ts_in[:b].copy_(G.ts)
        G.ts_in[b:].copy_(G.ts)
    else:
        G.lat_in.copy_(G.lat)
        G.ts_in.copy_(G.ts)
    unet.prepare_context(G.ctx)
    tape = []
    unet.forward(G.lat_in, G.ts_in, out=G.eps, tape=tape)
    eps = G.eps.view(G.nb, n)
    d_eps = G.d_eps.view(G.nb, n)
    if train_cfg:
        eu, ec, du, dc, g = eps[:b], eps[b:], d_eps[:b], d_eps[b:], float(guidance_scale)
    else:  # noise_pred = cond output: eps_u slot with guidance 0 reproduces it exactly
        eu, ec, du, dc, g = eps, eps, d_eps, None, 0.0
    x, nx = G.lat.view(b, n), G.nxt.view(b, n)
    ac = sched_state.common.alphas_cumprod
    fa = sched_state.final_alpha_cumprod
    ops.ddim_logprob_fwd(eu, ec, x, nx, ac, G.ts, fa, ratio, g, float(eta), G.logp, G.ws, pred=pred)
    ops.ppo_loss(G.logp, G.old_logp, G.adv, float(clip_range), G.info, G.dlogp, micro_batch=micro_batch or b)
    if dc is None:
        scratch = unet.arena.alloc((b, n), torch.float32)
        ops.ddim_logprob_bwd(eu, ec, x, nx, ac, G.ts, fa, ratio, g, float(eta), G.dlogp, du, scratch, G.ws, pred=pred)
        unet.arena.release(scratch)
    else:
        ops.ddim_logprob_bwd(eu, ec, x, nx, ac, G.ts, fa, ratio, g, float(eta), G.dlogp, du, dc, G.ws, pred=pred)
    unet.backward(tape, G.d_eps)


def train_step(state: AccumulatingTrainState, batch, noise_scheduler_state, noise_scheduler, train_cfg,
               guidance_scale, eta, clip_range, do_opt_update, micro_batch_size=None, pmean_info=True):
    """``micro_batch_size`` (extension, default = the batch size => exactly the reference call): the batch may
    stack several reference micro-batches -- e.g. the same ``train_batch_size`` samples at several of their
    timesteps, which the reference feeds through consecutive ``train_step`` calls at unchanged parameters
    (``pipeline/policy_gradient.py:410-441``) -- and is then processed as ONE large U-Net batch.  Gradients,
    ``n_acc`` and the averaged ``info`` equal those of the consecutive calls (up to fp32 summation order).

    ``pmean_info`` (extension, default True = the reference's ``lax.pmean(info)`` every call, :142): with False the returned
    ``info`` is this rank's; the epoch driver then averages the whole inner epoch's stack of infos over ranks in ONE
    collective (the mean is linear: same numbers) instead of synchronising every rank after every pass."""
    assert isinstance(state, AccumulatingTrainState)
    unet = state.apply_fn
    lat = batch["latents"]
    b = lat.shape[0]
    assert b == batch["ts"].shape[0] == batch["next_latents"].shape[0] == batch["log_probs"].shape[0]
    h, w = lat.shape[-2], lat.shape[-1]
    emb = batch["prompt_embeds"]
    key = (id(unet), b, h, w, tuple(emb.shape[1:]), bool(train_cfg))
    G = _GRAPHS.get(key)
    if G is None:
        G = _GRAPHS[key] = _StepGraph(unet, b, h, w, emb.shape[1], emb.shape[2], bool(train_cfg))
    G.lat.copy_(lat.reshape(b, 4, h, w))
    G.nxt.copy_(batch["next_latents"].reshape(b, 4, h, w))
    G.ts.copy_(torch.as_tensor(batch["ts"]).to(G.ts.device, torch.int32))
    G.old_logp.copy_(batch["log_probs"])
    G.adv.copy_(torch.as_tensor(batch["advantages"]).to(G.adv.device, torch.float32))
    if train_cfg:
        G.ctx[:b].copy_(batch["uncond_embeds"])
        G.ctx[b:].copy_(emb)
    else:
        G.ctx.copy_(emb)
    ratio = noise_scheduler.config.num_train_timesteps // noise_scheduler_state.num_inference_steps
    mb = int(micro_batch_size or b)
    assert b % mb == 0
    pred = noise_scheduler.config.prediction_type   # the reference branches on it inside scheduler.step (:303-321)
    sig = (float(guidance_scale), float(eta), float(clip_range), ratio, id(noise_scheduler_state.common.alphas_cumprod), mb, pred)

    def body():
        _run_body(unet, G, b, bool(train_cfg), noise_scheduler_state, ratio, guidance_scale, eta, clip_range, mb, pred)

    G.graph = graph_step(G.graph, sig, body, USE_CUDA_GRAPH, protect=state.grad_acc)
    info_t = G.info.clone()
    if pmean_info:
        distributed.pmean_(info_t)                                # lax.pmean(info) (:142)
    state.apply_gradients(grads=None, do_update=do_opt_update, n_micro=b // mb)
    info = {"approx_kl": info_t[0], "clipfrac": info_t[1], "loss": info_t[2]}
    return state, info


def smoke_train_step(unet, sched, state, lat, nxt, lps, ts, emb, neg):
    """Used by __graft_entry__.smoke(): one PPO step on a sampled trajectory; unchanged policy => ratio == 1."""
    ts_state = AccumulatingTrainState(apply_fn=unet)
    st = sched.set_timesteps(state, lat.shape[1])
    b = lat.shape[0]
    batch = {"latents": lat[:, 0].contiguous(), "next_latents": nxt[:, 0].contiguous(), "ts": ts[:, 0].contiguous(),
             "log_probs": lps[:, 0].contiguous(), "advantages": torch.tensor([1.0, -1.0][:b], device=lat.device),
             "prompt_embeds": emb.to(lat.device), "uncond_embeds": neg.to(lat.device)}
    _, info = train_step(ts_state, batch, st, sched, True, 5.0, 1.0, 1e-4, True)
    torch.cuda.synchronize()
    assert abs(info["approx_kl"].item()) == 0.0 and info["clipfrac"].item() == 0.0, info
