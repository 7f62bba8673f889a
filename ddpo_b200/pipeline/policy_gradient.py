"""DDPO epoch driver -- drop-in mirror of the reference's ``pipeline/policy_gradient.py`` (``main`` :44-480):
sample trajectories -> decode -> reward callbacks -> advantages -> shuffles -> PPO updates -> logs / checkpoints.

    python -m ddpo_b200.pipeline.policy_gradient --dataset compressed-animals [--key value ...]
    torchrun --nproc-per-node 8 -m ddpo_b200.pipeline.policy_gradient --dataset compressed-animals

Same config keys (``config/base.py`` "pg"), same host-side random streams (``np.random`` permutations in the same call
order, Python ``random`` prompts, the jax key lineage ``PRNGKey(seed) -> split -> per-batch split``), same log artefacts
(``args.json``, ``samples/*.png``, ``rewards|prompts|callback_info|per_prompt_stats|train_info/*.npy``,
``checkpoints/checkpoint_<epoch>``).

GPU design (SURVEY §8 a11/e):
  * one process per GPU (torchrun); a rank plays the role of one reference *worker* (``jax.process_index``) with one
    local device, so the per-worker batch permutation (:385-393) is already shard-local and no trajectory ever moves
    between GPUs; rewards / prompts are all-gathered exactly where the reference calls ``process_allgather``;
  * trajectories never leave HBM: the epoch keeps one ``[N, T+1, 4*h*w]`` buffer; the batch and per-sample time
    shuffles are realised as an index table consumed by a row-gather kernel (the reference round-trips 6.5 MB/sample
    through host NumPy and re-uploads a slice every step, :288-298, :415-423);
  * the ``train_macro`` consecutive timesteps of a minibatch -- which the reference feeds through that many
    ``train_step`` calls at unchanged parameters -- are ONE U-Net pass (``train_step(..., micro_batch_size=...)``);
    ``--train_macro 1`` reproduces the reference's call sequence one to one.
"""
import json
import os
import random
import time
from concurrent import futures

import numpy as np
import torch

from .. import ops, training, utils
from ..diffusers_patch import DDIMScheduler
from ..training import distributed
from ..training.policy_gradient import AccumulatingTrainState, AdafactorConfig, AdamWConfig, train_step
from ..utils.stat_tracking import PerPromptStatTracker


class Parser(utils.Parser):
    config = "ddpo_b200.config.base"
    dataset = "compressed_animals"


# ----------------------------------------------------------------- host logic ----
def set_seed(seed):
    """``transformers.set_seed`` (reference :46): Python, NumPy and torch generators."""
    random.seed(seed)
    np.random.seed(seed % (2 ** 32))
    torch.manual_seed(seed)


def batch_sizes(args, n_devices, process_count):
    """The derived sizes and the three divisibility asserts of reference :53-86."""
    train_worker = n_devices * args.train_batch_size
    train_pod = train_worker * process_count
    train_effective = train_pod * args.train_accumulation_steps
    sample_worker = n_devices * args.sample_batch_size
    sample_pod = sample_worker * process_count
    total = args.num_sample_batches_per_epoch * sample_pod
    assert args.sample_batch_size >= args.train_batch_size
    assert args.sample_batch_size % args.train_batch_size == 0
    assert total % train_effective == 0
    return dict(train_worker_batch_size=train_worker, train_pod_batch_size=train_pod,
                train_effective_batch_size=train_effective, sample_worker_batch_size=sample_worker,
                sample_pod_batch_size=sample_pod, total_samples_per_epoch=total,
                updates_per_inner_epoch=total // train_effective)


def compute_advantages(rewards, prompts, per_prompt_stats):
    """Reference :323-347: per-prompt tracker when configured, else the plain z-score (no epsilon)."""
    rewards = np.asarray(rewards)
    if per_prompt_stats is not None:
        return per_prompt_stats.update(np.asarray(prompts), rewards)
    return (rewards - np.mean(rewards)) / np.std(rewards)


def epoch_shuffles(total_batch_size, num_timesteps):
    """Reference :385-393, same ``np.random`` call order: one batch permutation, then an independent time
    permutation per (already permuted) sample."""
    perm = np.random.permutation(total_batch_size)
    perms = np.array([np.random.permutation(num_timesteps) for _ in range(total_batch_size)])
    return perm, perms


def pick_macro(num_train_ts, requested):
    """Largest divisor of ``num_train_ts`` that is <= ``requested`` (timesteps stacked into one U-Net pass)."""
    requested = max(1, min(int(requested), int(num_train_ts)))
    return max(d for d in range(1, requested + 1) if num_train_ts % d == 0)


def train_schedule(perm, perms, train_batch_size, num_train_ts, accumulation_steps, macro):
    """Yields one entry per U-Net training pass, in the reference's order (:410-441).

    Minibatch ``i`` holds the permuted rows ``k = i*B .. (i+1)*B-1``; the reference row ``k`` at shuffled time column
    ``j`` is the ORIGINAL sample ``perm[k]`` at original step ``perms[k, j]``.  Each entry covers columns
    ``j0 .. j0+J-1``: ``sample_idx [J*B]``, ``time_idx [J*B]`` (column-major: all B samples at j0, then at j0+1, ...),
    ``do_opt_update`` as :426-428 (true on the pass that contains the last trained column of every
    ``accumulation_steps``-th minibatch)."""
    total = len(perm)
    B = int(train_batch_size)
    assert total % B == 0 and num_train_ts % macro == 0
    for i in range(total // B):
        rows = np.arange(i * B, (i + 1) * B)
        for j0 in range(0, num_train_ts, macro):
            cols = np.arange(j0, j0 + macro)
            sample_idx = np.tile(perm[rows], macro)
            time_idx = perms[rows][:, cols].T.reshape(-1)
            last = (j0 + macro == num_train_ts) and ((i + 1) % accumulation_steps == 0)
            yield dict(i=i, j0=j0, J=macro, rows=rows, sample_idx=sample_idx, time_idx=time_idx, do_opt_update=last)


def allgather_array(x):
    """``multihost_utils.process_allgather(x, tiled=True)``: concatenate over workers along axis 0."""
    x = np.asarray(x)
    w = distributed.world_size()
    if w == 1:
        return x
    if x.dtype.kind in "fiu":
        # numeric arrays (rewards, prompt ids): one tensor all_gather -- every worker holds the same shape (the reference
        # shards batches evenly) -- instead of pickling through all_gather_object
        dev = torch.device("cuda", torch.cuda.current_device()) if torch.distributed.get_backend() == "nccl" else "cpu"
        t = torch.from_numpy(np.ascontiguousarray(x)).to(dev)
        out = [torch.empty_like(t) for _ in range(w)]
        torch.distributed.all_gather(out, t)
        return np.concatenate([o.cpu().numpy() for o in out])
    out = [None] * w
    torch.distributed.all_gather_object(out, x)
    return np.concatenate(out)


# ------------------------------------------------------------- device-side data ----
class EpochBuffer:
    """The epoch's trajectories in HBM: ``traj [N, T+1, n]`` (row (s, t) = x_t of sample s; ``latents`` = rows t<T,
    ``next_latents`` = rows t+1), ``embeds [N, L, D]``; small per-step scalars stay on the host as the reference's
    ``samples`` dict does (``log_probs [N, T]``, ``ts [N, T]``)."""

    def __init__(self, n_samples, T, lat_shape, ctx_shape, device):
        self.N, self.T = n_samples, T
        self.lat_shape = tuple(lat_shape)
        self.n = int(np.prod(lat_shape))
        self.traj = torch.empty(n_samples, T + 1, self.n, device=device)
        self.embeds = torch.empty(n_samples, *ctx_shape, device=device)
        self.log_probs = np.empty((n_samples, T), np.float32)
        self.ts = np.empty((n_samples, T), np.int32)
        self.filled = 0

    def append(self, final_latents, latents, log_probs, ts, embeds):
        b = final_latents.shape[0]
        s = slice(self.filled, self.filled + b)
        self.traj[s, : self.T].copy_(latents.reshape(b, self.T, self.n))
        self.traj[s, self.T].copy_(final_latents.reshape(b, self.n))
        self.embeds[s].copy_(embeds)
        self.log_probs[s] = log_probs.detach().float().cpu().numpy()
        self.ts[s] = ts.detach().cpu().numpy()
        self.filled += b

    def gather(self, sample_idx, time_idx, advantages, uncond_row):
        """Builds the ``train_step`` batch of :415-423 for the given (sample, time) rows, all on the device."""
        dev = self.traj.device
        rows = len(sample_idx)
        flat_idx = np.asarray(sample_idx, np.int64) * (self.T + 1) + np.asarray(time_idx, np.int64)
        idx = torch.from_numpy(np.concatenate([flat_idx, flat_idx + 1, np.asarray(sample_idx, np.int64)])).to(dev)
        lat = torch.empty(rows, *self.lat_shape, device=dev)
        nxt = torch.empty(rows, *self.lat_shape, device=dev)
        emb = torch.empty(rows, *self.embeds.shape[1:], device=dev)
        table = self.traj.view(self.N * (self.T + 1), self.n)
        ops.gather_rows(table, idx[:rows], lat.view(rows, self.n))
        ops.gather_rows(table, idx[rows:2 * rows], nxt.view(rows, self.n))
        ops.gather_rows(self.embeds.view(self.N, -1), idx[2 * rows:], emb.view(rows, -1))
        host = np.stack([self.log_probs[sample_idx, time_idx], np.asarray(advantages, np.float32)[sample_idx]])
        hd = torch.from_numpy(host.astype(np.float32)).to(dev)
        ts = torch.from_numpy(self.ts[sample_idx, time_idx].astype(np.int32)).to(dev)
        return {"prompt_embeds": emb, "uncond_embeds": uncond_row.expand(rows, -1, -1), "advantages": hd[1],
                "latents": lat, "next_latents": nxt, "log_probs": hd[0], "ts": ts}


class _nvtx:
    """NVTX range per phase of the epoch loop (sample / decode / reward wait / train / optimizer update) so that a timeline
    capture of the driver reads like the reference's loop; a no-op without CUDA."""

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if torch.cuda.is_available():
            torch.cuda.nvtx.range_push(self.name)

    def __exit__(self, *exc):
        if torch.cuda.is_available():
            torch.cuda.nvtx.range_pop()


def vae_decode(pipeline, final_latents):
    """Reference :174-182 (``latents / 0.18215`` -> VAE decoder -> ``(x/2+.5).clip(0,1)`` NHWC float32)."""
    if pipeline.vae is None:
        raise RuntimeError("the pipeline has no VAE decoder attached (utils.load_unet(with_vae=True))")
    return pipeline.vae.decode_to_images(final_latents)


def save_png(path, image):
    from PIL import Image
    image = np.asarray(image)
    if image.dtype != np.uint8:
        image = (np.clip(image, 0, 1) * 255).round().astype("uint8")
    Image.fromarray(image).save(path)


def images_to_host(images, as_uint8):
    """decoded images [N,H,W,3] in [0,1] (device, fp32) -> host array.  ``as_uint8``: the reference's
    ``(image * 255).astype(np.uint8)`` (callbacks.py:181) runs on the device and the bytes go through pinned memory --
    6 MB instead of 25 MB per 8 images; rewards that take floats get the fp32 array as before (:275)."""
    if as_uint8:
        u8 = torch.empty(images.shape, dtype=torch.uint8, device=images.device)
        ops.image_to_uint8(images.contiguous(), u8)
        if not images.is_cuda:   # CPU dry run of the host logic on the test suite's ops emulator
            return u8.numpy()
        host = torch.empty(images.shape, dtype=torch.uint8, pin_memory=True)
        host.copy_(u8)
        return host.numpy()
    return images.detach().float().cpu().numpy()


# ------------------------------------------------------------------------ main ----
def main(argv=None, models=None, max_epochs=None, save_last=True):
    """``models``: optional ``(pipeline, params)`` (tests / bench inject a random-init model); ``max_epochs`` caps
    ``num_train_epochs``; ``save_last=False`` skips the unconditional checkpoint of the final epoch (bench: a
    3.5 GB file).  Returns a dict of per-epoch statistics."""
    args = Parser().parse_args("pg", argv)
    if not hasattr(args, "train_macro"):
        args.train_macro = 10
    set_seed(args.seed)
    worker_id, process_count, n_devices = distributed.rank(), distributed.world_size(), 1
    if torch.cuda.is_available():
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    # no CUDA device: the kernels refuse CPU tensors (ops._p), so this only serves the CPU dry run of the host logic
    # on the test suite's ops emulator (tests/test_drivers_host_cpu.py)
    device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")

    rng = ops.prng_key(args.seed)                                                   # :51
    sizes = batch_sizes(args, n_devices, process_count)
    print(f"[ policy_gradient ] local devices: {n_devices} | number of workers: {process_count}")
    print(f"[ policy_gradient ] sample worker batch size: {sizes['sample_worker_batch_size']} | "
          f"sample pod batch size: {sizes['sample_pod_batch_size']}")
    print(f"[ policy_gradient ] train worker batch size: {sizes['train_worker_batch_size']} | "
          f"train pod batch size: {sizes['train_pod_batch_size']} | "
          f"train accumulated batch size: {sizes['train_effective_batch_size']}")
    print(f"[ policy_gradient ] number of sample batches per epoch: {args.num_sample_batches_per_epoch}")
    print(f"[ policy_gradient ] total number of samples per epoch: {sizes['total_samples_per_epoch']}")
    print(f"[ policy_gradient ] number of gradient updates per inner epoch: {sizes['updates_per_inner_epoch']}")

    localpath = "logs/" + args.savepath.replace("gs://", "")                        # :90
    os.makedirs(localpath, exist_ok=True)
    with open(f"{localpath}/args.json", "w") as f:
        json.dump(args._dict, f, indent=4, default=str)

    # --------------------------------- models ---------------------------------#
    print("loading models...")
    if models is None:
        models = utils.load_unet(args.loadpath or None, epoch=args.load_epoch, pretrained_model=args.pretrained_model,
                                 dtype=args.dtype, cache=args.cache, device=device)
    pipeline, params = models
    pipeline.safety_checker = None
    c = pipeline.scheduler.config
    pipeline.scheduler = DDIMScheduler(num_train_timesteps=c.num_train_timesteps, beta_start=c.beta_start,   # :107-116
                                       beta_end=c.beta_end, beta_schedule=c.beta_schedule,
                                       trained_betas=c.trained_betas, set_alpha_to_one=c.set_alpha_to_one,
                                       steps_offset=c.steps_offset, prediction_type=c.prediction_type, device=device)
    cfg = pipeline.unet.cfg
    lat_hw = args.resolution // pipeline.vae_scale_factor
    noise_scheduler_state = pipeline.scheduler.set_timesteps(                                             # :117-126
        params["scheduler"], num_inference_steps=args.n_inference_steps,
        shape=(args.train_batch_size, cfg.in_channels, lat_hw, lat_hw))

    # ------------------------------- optimizer --------------------------------#
    print("initializing train state...")
    optimizers = {                                                                                         # :130-150
        "adamw": lambda: AdamWConfig(learning_rate=args.learning_rate, b1=args.beta1, b2=args.beta2, eps=args.epsilon,
                                     weight_decay=args.weight_decay, max_grad_norm=args.max_grad_norm),
        "adafactor": lambda: AdafactorConfig(learning_rate=args.learning_rate, weight_decay=args.weight_decay,
                                             max_grad_norm=args.max_grad_norm),
    }
    if args.optimizer not in optimizers:
        raise ValueError(f"optimizer={args.optimizer!r}: must be one of {', '.join(optimizers)}")
    tx = optimizers[args.optimizer]()
    lora_rank = int(getattr(args, "lora_rank", 0) or 0)
    if lora_rank:   # adapters on the attention projections, the U-Net frozen; args.seed carries + rank (utils/parser.py):
        pipeline.unet.enable_lora(lora_rank, seed=args.seed - worker_id)   # every rank builds the same adapters
    state = AccumulatingTrainState(step=0, apply_fn=pipeline.unet, params=params["unet"], tx=tx, n_acc=0)  # :156-164

    timer = utils.Timer()

    def text_encode(input_ids):                                                                            # :185-187
        out = pipeline.text_encoder(input_ids, params=params.get("text_encoder"))
        out = out[0] if isinstance(out, (tuple, list)) else out
        return torch.as_tensor(np.asarray(out, np.float32)) if not torch.is_tensor(out) else out.float()

    uncond_ids = pipeline.prepare_inputs([""])                                                             # :190
    timer()
    uncond_prompt_embeds = text_encode(uncond_ids).to(device)                                              # [1, L, D]
    print(f"[ embed uncond prompts ] in {timer():.2f}s")
    sample_uncond = uncond_prompt_embeds.expand(args.sample_batch_size, -1, -1).contiguous()               # :195-199

    train_rng, sample_rng = ops.threefry_split(rng, 2)                                                     # :201
    callback_fns = {args.filter_field: training.callback_fns[args.filter_field]()}                        # :204-206
    uint8_images = all(getattr(f, "accepts_uint8", False) for f in callback_fns.values())
    executor = futures.ThreadPoolExecutor(max_workers=2)                                                   # :211
    per_prompt_stats = None
    if args.per_prompt_stats_bufsize is not None:
        per_prompt_stats = PerPromptStatTracker(args.per_prompt_stats_bufsize, args.per_prompt_stats_min_count)

    T = args.n_inference_steps
    n_local = args.num_sample_batches_per_epoch * n_devices * args.sample_batch_size
    mean_rewards, std_rewards, history = [], [], []
    n_epochs = args.num_train_epochs if max_epochs is None else min(args.num_train_epochs, max_epochs)
    for epoch in range(n_epochs):
        t_epoch = time.time()
        buf = EpochBuffer(n_local, T, (cfg.in_channels, lat_hw, lat_hw), (cfg.ctx_len, cfg.cross_attention_dim), device)
        all_prompts, pending = [], []
        for i in range(args.num_sample_batches_per_epoch):
            sample_prompts, training_prompts, prompt_metadata = training.make_prompts(                     # :236-242
                args.prompt_fn, n_devices * args.sample_batch_size, args.identical_batch, evaluate=args.evaluate,
                **args.prompt_kwargs)
            sample_rng, sample_seed = ops.threefry_split(sample_rng, 2)                                    # :244
            sample_seeds = ops.threefry_split(sample_seed, n_devices)                                      # :245
            sample_prompt_ids = pipeline.prepare_inputs(sample_prompts)
            sample_prompt_embeds = text_encode(sample_prompt_ids).to(device)
            timer()
            sampling_params = {"unet": state.params, "scheduler": params["scheduler"]}
            with _nvtx(f"ddpo/sample e{epoch} b{i}"):
                final_latents, latents, next_latents, log_probs, ts = pipeline(                            # :256-268
                    sample_prompt_embeds, sample_uncond, sampling_params, sample_seeds[0], T, jit=True,
                    height=args.resolution, width=args.resolution, guidance_scale=args.guidance_scale, eta=args.eta)
            with _nvtx("ddpo/vae_decode"):
                images = vae_decode(pipeline, final_latents)                                               # :271
            images = images_to_host(images, uint8_images)                                                 # :275
            callbacks = executor.submit(training.evaluate_callbacks, callback_fns, images, sample_prompts,
                                        prompt_metadata)                                                   # :277-283
            time.sleep(0)
            buf.append(final_latents, latents, log_probs, ts, sample_prompt_embeds)                        # :288-298
            all_prompts += list(sample_prompts)
            pending.append(callbacks)
            save_png(utils.fs.join_and_create(localpath, f"samples/{worker_id}_{epoch}_{i}.png"), images[0])  # :301

        rewards_l, info_l = [], []
        for cb in pending:                                                                                 # :312-316
            r, info = cb.result()[args.filter_field]
            rewards_l.append(np.asarray(r))
            info_l.append(info)
        local_rewards = np.concatenate(rewards_l)
        rewards = np.array(allgather_array(local_rewards))                                                 # :323-325
        local_prompts = np.array(all_prompts)
        if per_prompt_stats is not None:                                                                   # :328-345
            prompt_ids = pipeline.tokenizer(local_prompts.tolist(), padding="max_length", return_tensors="np").input_ids
            prompt_ids = allgather_array(prompt_ids)
            prompts = np.array(pipeline.tokenizer.batch_decode(prompt_ids, skip_special_tokens=True))
            advantages = per_prompt_stats.update(prompts, rewards)
            if worker_id == 0:
                np.save(utils.fs.join_and_create(localpath, f"per_prompt_stats/{worker_id}_{epoch}.npy"),
                        per_prompt_stats.get_stats())
        else:
            advantages = (rewards - np.mean(rewards)) / np.std(rewards)                                    # :347
        advantages = np.asarray(advantages).reshape(process_count, -1)[worker_id]                          # :349
        advantages = advantages.reshape(-1)
        print(f"mean reward: {np.mean(rewards):.4f}")
        mean_rewards.append(float(np.mean(rewards)))
        std_rewards.append(float(np.std(rewards)))
        np.save(utils.fs.join_and_create(localpath, f"rewards/{worker_id}_{epoch}.npy"), local_rewards)    # :356-369
        np.save(utils.fs.join_and_create(localpath, f"prompts/{worker_id}_{epoch}.npy"), local_prompts)
        np.save(utils.fs.join_and_create(localpath, f"callback_info/{worker_id}_{epoch}.npy"),
                np.array(info_l, dtype=object), allow_pickle=True)
        t_sample = time.time() - t_epoch

        t_train0 = time.time()
        epoch_infos = []
        for inner_epoch in range(args.num_inner_epochs):                                                   # :375-455
            total_batch_size, num_timesteps = buf.log_probs.shape
            assert total_batch_size == n_local and num_timesteps == T
            perm, perms = epoch_shuffles(total_batch_size, num_timesteps)
            num_train_ts = int(num_timesteps * args.train_timestep_ratio)
            macro = pick_macro(num_train_ts, args.train_macro)
            all_infos, do_opt_update = [], False
            for step in train_schedule(perm, perms, args.train_batch_size, num_train_ts,
                                       args.train_accumulation_steps, macro):
                batch = buf.gather(step["sample_idx"], step["time_idx"], advantages, uncond_prompt_embeds)
                do_opt_update = step["do_opt_update"]
                if do_opt_update:
                    print(f"opt update at {step['i']}, {step['j0'] + macro - 1}")
                with _nvtx("ddpo/train_step+update" if do_opt_update else "ddpo/train_step"):
                    state, info = train_step(state, batch, noise_scheduler_state, pipeline.scheduler, args.train_cfg,
                                             args.guidance_scale, args.eta, args.ppo_clip_range, do_opt_update,
                                             micro_batch_size=args.train_batch_size, pmean_info=False)
                all_infos.append(info)
            assert do_opt_update                                                                           # :446
            # lax.pmean(info) (reference training/policy_gradient.py:142) for the whole inner epoch in one collective
            keys = list(all_infos[0])
            stacked = torch.stack([torch.stack([i[k] for k in keys]) for i in all_infos])                  # [steps, 3]
            distributed.pmean_(stacked)
            stacked = stacked.cpu().numpy()
            all_infos = {k: stacked[:, j].astype(np.float64) for j, k in enumerate(keys)}
            print(f"mean info: { {k: float(np.mean(v)) for k, v in all_infos.items()} }")
            if worker_id == 0:
                np.save(utils.fs.join_and_create(localpath, f"train_info/{worker_id}_{epoch}_{inner_epoch}.npy"),
                        all_infos)
            epoch_infos.append(all_infos)
        if torch.cuda.is_available():
            torch.cuda.synchronize()
        t_train = time.time() - t_train0

        if (epoch + 1) % args.save_freq == 0 or (epoch == n_epochs - 1 and save_last):                     # :457-464
            # LoRA mode: the checkpoint holds the merged U-Net (W + D U), so that its readers see a fine-tuned U-Net
            flat = pipeline.unet.merged_params() if lora_rank else state.params
            utils.save_checkpoint_multiprocess(os.path.join(args.savepath, "checkpoints"),
                                               utils.params_tree(flat, cfg), step=epoch, keep=1e6, overwrite=True)
        history.append(dict(epoch=epoch, mean_reward=mean_rewards[-1], std_reward=std_rewards[-1],
                            sample_seconds=t_sample, train_seconds=t_train, infos=epoch_infos,
                            samples=sizes["total_samples_per_epoch"]))
        if worker_id == 0:
            try:                                                                                           # :467-478
                import matplotlib.pyplot as plt
                plt.clf()
                plt.plot(mean_rewards, color="black")
                plt.savefig(os.path.join(localpath, f"log_{worker_id}.png"))
            except ImportError:
                np.save(os.path.join(localpath, f"log_{worker_id}.npy"), np.array([mean_rewards, std_rewards]))
    executor.shutdown()
    return dict(history=history, state=state, localpath=localpath)


if __name__ == "__main__":
    if "RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1:
        torch.distributed.init_process_group("nccl" if torch.cuda.is_available() else "gloo")
    main()
