#!/usr/bin/env python
"""Full fine-tuning vs. LoRA rank 4 (``UNet.enable_lora``) at the bench configuration: random-init SD2-base, 512 px,
a PPO train pass of 10 timesteps x train batch 2 with CFG (U-Net fwd + bwd at batch 40), and one optimizer update
(AdamW).  The arms alternate (full, LoRA, full, LoRA, ...) in one process, each on a freshly built U-Net.

    python tests/bench_lora.py [--rounds 2] [--steps 5] [--updates 3]

Prints the card and its power limit, per arm ms per train pass and per update (median and spread over the timed
calls), peak device memory, and per adapter-gradient launch (ops.lora_grad) its CUDA-event time and achieved GB/s
against its minimum bytes (x and every dy read once), as a fraction of 3.35 TB/s."""
import argparse
import gc
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ddpo_b200 import ops, unet_spec as S  # noqa: E402
from ddpo_b200.diffusers_patch import DDIMScheduler  # noqa: E402
from ddpo_b200.training import policy_gradient as pg  # noqa: E402
from ddpo_b200.unet import UNet  # noqa: E402

HBM_TBS = 3.35


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:   # noqa: BLE001
        pl = "unknown"
    return name, pl


def make_batch(dev, bt=2, j=10, seed=0):
    g = torch.Generator().manual_seed(seed)
    n = bt * j
    return {"latents": torch.randn(n, 4, 64, 64, generator=g).to(dev),
            "next_latents": torch.randn(n, 4, 64, 64, generator=g).to(dev),
            "ts": torch.tensor([981 - 20 * (i // bt) for i in range(n)], dtype=torch.int32, device=dev),
            "log_probs": torch.zeros(n, device=dev), "advantages": torch.tensor([1.0, -1.0] * j, device=dev),
            "prompt_embeds": torch.randn(n, 77, 1024, generator=g).to(dev),
            "uncond_embeds": torch.randn(1, 77, 1024, generator=g).expand(n, -1, -1).contiguous().to(dev)}


def run_arm(lora, flat, args, dev):
    torch.cuda.reset_peak_memory_stats()
    net = UNet(S.SD2_BASE, flat, dev)
    if lora:
        net.enable_lora(4, seed=0)
    tstate = pg.AccumulatingTrainState(apply_fn=net)
    sched = DDIMScheduler(1000, 0.00085, 0.012, "scaled_linear", None, False, 1, "epsilon", device=dev)
    st = sched.set_timesteps(sched.create_state(), 50)
    batch = make_batch(dev)
    step = lambda upd: pg.train_step(tstate, batch, st, sched, True, 5.0, 1.0, 1e-4, upd, micro_batch_size=2,  # noqa: E731
                                     pmean_info=False)
    for _ in range(3):
        step(False)
    torch.cuda.synchronize()

    def timed(upd):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step(upd)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)
    passes = [timed(False) for _ in range(args.steps)]
    with_update = [timed(True) for _ in range(args.updates)]
    mp = float(np.median(passes))
    updates = [t - mp for t in with_update]
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    launches = []
    if lora:    # one eager pass with CUDA events around every launch
        pg.USE_CUDA_GRAPH = False
        ops.PROFILE, ops.PROFILE_TAGS[:] = [], []
        step(False)
        torch.cuda.synchronize()
        for (name, work, e0, e1), tag in zip(ops.PROFILE, ops.PROFILE_TAGS):
            if name == "lora_grad":
                ms = e0.elapsed_time(e1)
                launches.append((tag, ms, work / ms / 1e6))
        ops.PROFILE = None
        pg.USE_CUDA_GRAPH = True
    del tstate, net
    pg._GRAPHS.clear()
    gc.collect()
    torch.cuda.empty_cache()
    return dict(passes=passes, updates=updates, peak_gib=peak, launches=launches)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--updates", type=int, default=3)
    args = ap.parse_args()
    dev = "cuda"
    name, pl = card()
    print(f"card: {name} | power limit: {pl}")
    flat = S.init_flat_params(S.SD2_BASE, 0)
    res = {"full": [], "lora4": []}
    for r in range(args.rounds):
        for arm in ("full", "lora4"):
            out = run_arm(arm == "lora4", flat, args, dev)
            res[arm].append(out)
            print(f"round {r} {arm:5s}: train pass {np.median(out['passes']):8.1f} ms "
                  f"[{min(out['passes']):.1f}, {max(out['passes']):.1f}] | update {np.median(out['updates']):7.1f} ms "
                  f"[{min(out['updates']):.1f}, {max(out['updates']):.1f}] | peak {out['peak_gib']:.2f} GiB", flush=True)
    summary = {}
    for arm, outs in res.items():
        p = [t for o in outs for t in o["passes"]]
        u = [t for o in outs for t in o["updates"]]
        summary[arm] = dict(pass_ms=float(np.median(p)), pass_min=float(min(p)), pass_max=float(max(p)),
                            update_ms=float(np.median(u)), update_min=float(min(u)), update_max=float(max(u)),
                            peak_gib=max(o["peak_gib"] for o in outs))
    launches = res["lora4"][-1]["launches"]
    print(f"adapter-gradient launches of one pass: {len(launches)}, {sum(ms for _, ms, _ in launches):.2f} ms in all")
    agg = {}
    for tag, ms, gbs in launches:
        agg.setdefault(tag, []).append((ms, gbs))
    for tag, v in sorted(agg.items()):
        ms = np.median([a for a, _ in v])
        gbs = np.median([b for _, b in v])
        print(f"  {tag:32s} x{len(v):2d}: {ms * 1e3:8.1f} us  {gbs:7.1f} GB/s  ({gbs / (HBM_TBS * 1e3) * 100:5.1f} % of "
              f"{HBM_TBS} TB/s)")
    print(json.dumps(dict(card=name, power_limit=pl, **summary)))


if __name__ == "__main__":
    main()
