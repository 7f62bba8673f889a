"""The optimizer update on one GPU: clip + AdamW against clip + Adafactor on the SD2-base and SD1 flat buffers.

    python tests/bench_optim.py [--seconds 1.5] [--out results/bench_optim.json]

Prints the card name and power limit first, then per model:
- ms per update of grad_sumsq + clip_adamw and of grad_sumsq + clip_adafactor, timed with CUDA events after warm-up
  over at least --seconds of back-to-back updates, with the bytes each moves by count, GB/s and the share of the
  H100 SXM data-sheet 3.35 TB/s.  Bytes per parameter: the norm pass reads g (4); clip_adamw reads g, p, nu, mu and
  writes p, nu, mu, g (28); clip_adafactor reads g and p in its statistics pass (8), g again for sum u^2 (4) and
  g and p in its apply pass, writing p and g (16), plus its tile partials and state;
- the time of each Adafactor kernel, from a torch.profiler run of its own after the timed runs;
- peak device memory of one bench-sized train pass (U-Net forward + backward at batch 40, 64 x 64 latents) followed by
  one optimizer update, with the train state built first as the DDPO driver builds it, under each optimizer.
"""
import argparse
import json
import math
import os
import re
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

DEV = "cuda"
HBM = 3.35e12
TRAIN_B = 40


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "unknown"
    return f"{name}, power limit / max SM clock: {q}"


def time_ms(fn, seconds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    iters = max(10, math.ceil(seconds * 1e3 / max(e0.elapsed_time(e1), 1e-3)))
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, iters


def updates(name, seconds):
    from ddpo_b200 import ops, unet_spec
    cfg = getattr(unet_spec, name)
    table, n = unet_spec.param_offsets(cfg)
    plan = ops.adafactor_plan(list(table.values()), n)
    gen = torch.Generator(device=DEV).manual_seed(0)
    p = torch.randn(n, device=DEV, generator=gen) * 0.05
    g = torch.randn(n, device=DEV, generator=gen) * 1e-5
    ws, sumsq = ops.optim_workspace(p.device), torch.zeros(1, device=DEV)
    res = {"model": name, "params": n}
    mu, nu = torch.zeros(n, dtype=torch.bfloat16, device=DEV), torch.zeros(n, device=DEV)

    def adamw():
        ops.grad_sumsq(g, ws, sumsq)
        ops.clip_adamw(p, g, mu, nu, sumsq, 1.0, 1.0, 1e-5, 0.9, 0.999, 1e-8, 1e-4, 1)
    res["adamw_ms"], res["adamw_iters"] = time_ms(adamw, seconds)
    res["adamw_bytes"] = 32.0 * n
    del mu, nu
    state = torch.zeros(plan.state_floats, device=DEV)
    aws = torch.zeros(plan.workspace_floats, device=DEV)
    parts = int((plan.tiles[:, 8] >= 0).sum()) * 256

    def adafactor():
        ops.grad_sumsq(g, ws, sumsq)
        ops.clip_adafactor(p, g, state, plan, aws, sumsq, 1.0, 1.0, 1e-5, 1e-4, 1)
    res["adafactor_ms"], res["adafactor_iters"] = time_ms(adafactor, seconds)
    # norm 4 + stats 8 + u^2 4 + apply 16 per parameter; tile partials written once and read once; state read and
    # written in the statistics pass and read twice more
    res["adafactor_bytes"] = 32.0 * n + 8.0 * parts + 16.0 * plan.state_floats
    for k in ("adamw", "adafactor"):
        res[f"{k}_gbs"] = res[f"{k}_bytes"] / (res[f"{k}_ms"] * 1e-3) / 1e9
        res[f"{k}_hbm_share"] = res[f"{k}_gbs"] * 1e9 / HBM
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            adafactor()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        m = re.search(r"\b(af_\w+_kernel|sumsq_\w+_kernel)", e.key)
        if m:
            kern[m.group(1)] = e.device_time_total / max(e.count, 1) / 1e3   # ms per launch
    res["adafactor_kernels_ms"] = kern
    return res


def train_peak(optimizer):
    from ddpo_b200 import unet_spec
    from ddpo_b200.training import policy_gradient as pg
    from ddpo_b200.unet import UNet
    cfg = unet_spec.SD2_BASE
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    net = UNet(cfg, unet_spec.init_flat_params(cfg, 0), DEV)
    tx = pg.AdafactorConfig() if optimizer == "adafactor" else pg.AdamWConfig()
    state = pg.AccumulatingTrainState(apply_fn=net, tx=tx)
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(TRAIN_B, 4, 64, 64, generator=g).to(DEV)
    ctx = torch.randn(TRAIN_B, 77, cfg.cross_attention_dim, generator=g).to(DEV)
    ts = torch.randint(1, 1000, (TRAIN_B,), generator=g, dtype=torch.int32).to(DEV)
    d_eps = (torch.randn(TRAIN_B, 4, 64, 64, generator=g) / (4 * 64 * 64)).to(DEV)
    net.prepare_context(ctx)
    tape = []
    net.forward(lat, ts, tape=tape)
    net.backward(tape, d_eps)
    state.apply_gradients(do_update=True)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 1e9
    del net, state, tape
    torch.cuda.empty_cache()
    return peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_optim measures on a CUDA device"
    result = {"card": card(), "updates": [], "train_peak_gb": {}}
    print(result["card"], flush=True)
    for name in ("SD2_BASE", "SD1"):
        r = updates(name, args.seconds)
        result["updates"].append(r)
        for k in ("adamw", "adafactor"):
            print(f"{name} {k}: {r[k + '_ms']:.2f} ms per update ({r[k + '_iters']} updates), "
                  f"{r[k + '_bytes'] / r['params']:.2f} B/param, {r[k + '_gbs']:.0f} GB/s, "
                  f"{100 * r[k + '_hbm_share']:.1f}% of 3.35 TB/s", flush=True)
        print(f"{name} adafactor kernels (ms per launch): "
              + ", ".join(f"{k} {v:.3f}" for k, v in r["adafactor_kernels_ms"].items()), flush=True)
    for opt in ("adamw", "adafactor", "adafactor", "adamw"):
        peak = train_peak(opt)
        result["train_peak_gb"].setdefault(opt, []).append(peak)
        print(f"SD2-base train pass (batch {TRAIN_B}) + one {opt} update: peak {peak:.2f} GB", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
