"""SD1.x against SD2-base on one GPU: attention kernels per head dim and whole U-Net passes.

    python tests/bench_sd1.py [--iters 20] [--rounds 2] [--out results/bench_sd1.json]

Prints the card name and power limit first, then:
- attention forward (sampling, batch 16) and forward + backward (training, batch 40) at the shapes each U-Net runs:
  self-attention at every level and cross-attention with Nk = 77.  SD1 has 8 heads everywhere (d = 40, 80, 160);
  SD2-base has d = 64 (5, 10, 20 heads).  TFLOP/s count the algorithmic FLOPs with the real head dim:
  forward 4 B h Nq Nk d (Q K^T and P V), backward 10 B h Nq Nk d (S recomputed, dP, dV, dK, dQ);
- ms per U-Net forward at batch 16 (one CFG denoising step of 8 samples: the U-Net part of a bench.py sampling step)
  and per U-Net forward + backward at batch 40 (one train pass: train batch 2 x train_macro 10, bench.py's PPO pass
  without the DDIM log-prob and loss kernels), with the peak device memory of each model.  The models are built one
  at a time (both at once would not fit) and alternate SD1, SD2, SD2, SD1, ...
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

DEV = "cuda"
SAMPLE_B, TRAIN_B = 16, 40
# (level tokens, SD1 heads x d, SD2 heads x d): the transformer levels of a 64 x 64 latent
LEVELS = [(4096, (8, 40), (5, 64)), (1024, (8, 80), (10, 64)), (256, (8, 160), (20, 64)), (64, (8, 160), (20, 64))]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "unknown"
    return f"{name}, power limit / max SM clock: {q}"


def time_ms(fn, iters, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def attention_case(b, heads, d, nq, nk, backward, iters):
    from ddpo_b200 import ops
    c = heads * d
    g = torch.Generator(device="cpu").manual_seed(0)
    if nk == nq:   # self: q/k/v are column slices of one [b n, 3C] buffer
        qkv = torch.randn(b * nq, 3 * c, generator=g).to(torch.bfloat16).to(DEV)
        q, k, v, ldq, ldk = qkv, qkv[:, c:], qkv[:, 2 * c:], 3 * c, 3 * c
    else:          # cross: q [b n, C], k/v slices of the [b 77, 2C] context projection
        q = torch.randn(b * nq, c, generator=g).to(torch.bfloat16).to(DEV)
        kv = torch.randn(b * nk, 2 * c, generator=g).to(torch.bfloat16).to(DEV)
        k, v, ldq, ldk = kv, kv[:, c:], c, 2 * c
    out = torch.empty(b * nq, c, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(b, heads, nq, device=DEV)
    fwd = lambda: ops.attention_fwd(q, k, v, out, b, heads, nq, nk, ldq, ldk, ldk, c, lse=lse, head_dim=d)
    res = {"fwd_ms": time_ms(fwd, iters)}
    res["fwd_tflops"] = 4.0 * b * heads * nq * nk * d / (res["fwd_ms"] * 1e-3) / 1e12
    if backward:
        do = torch.randn(b * nq, c, generator=g).to(torch.bfloat16).to(DEV)
        dq = torch.empty(b * nq, c, dtype=torch.bfloat16, device=DEV)
        dkv = torch.empty(b * nk, 2 * c, dtype=torch.bfloat16, device=DEV)
        delta = torch.empty(b, heads, nq, device=DEV)
        bwd = lambda: ops.attention_bwd(q, k, v, out, do, lse, delta, dq, dkv, dkv[:, c:], b, heads, nq, nk, ldq, ldk, ldk, c,
                                        c, c, 2 * c, 2 * c, head_dim=d)
        res["bwd_ms"] = time_ms(bwd, iters)
        res["bwd_tflops"] = 10.0 * b * heads * nq * nk * d / (res["bwd_ms"] * 1e-3) / 1e12
    return res


def unet_passes(name, iters):
    from ddpo_b200 import unet_spec
    from ddpo_b200.unet import UNet
    cfg = getattr(unet_spec, name)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    net = UNet(cfg, unet_spec.init_flat_params(cfg, 0), DEV)
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(TRAIN_B, 4, 64, 64, generator=g).to(DEV)
    ctx = torch.randn(TRAIN_B, 77, cfg.cross_attention_dim, generator=g).to(DEV)
    ts = torch.randint(1, 1000, (TRAIN_B,), generator=g, dtype=torch.int32).to(DEV)
    d_eps = (torch.randn(TRAIN_B, 4, 64, 64, generator=g) / (4 * 64 * 64)).to(DEV)
    net.prepare_context(ctx[:SAMPLE_B])
    fwd_ms = time_ms(lambda: net.forward(lat[:SAMPLE_B], ts[:1]), iters)
    net.enable_training()
    net.prepare_context(ctx)

    def train():
        tape = []
        net.forward(lat, ts, tape=tape)
        net.backward(tape, d_eps)
    train_ms = time_ms(train, max(2, iters // 4), warm=2)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    del net
    torch.cuda.empty_cache()
    return {"model": name, "unet_fwd_b16_ms": fwd_ms, "unet_fwd_bwd_b40_ms": train_ms, "peak_gib": peak}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sd1 measures on a CUDA device"
    result = {"card": card(), "attention": [], "unet": []}
    print(result["card"], flush=True)
    for n, sd1, sd2 in LEVELS:
        for model, (heads, d) in (("SD1", sd1), ("SD2", sd2)):
            for nk in (n, 77):
                for b, bwd in ((SAMPLE_B, False), (TRAIN_B, True)):
                    r = attention_case(b, heads, d, n, nk, bwd, args.iters)
                    r.update(model=model, batch=b, heads=heads, d=d, nq=n, nk=nk)
                    result["attention"].append(r)
                    line = (f"attention {model} b{b} h{heads} d{d} nq{n} nk{nk}: fwd {r['fwd_ms']:.3f} ms "
                            f"{r['fwd_tflops']:.1f} TFLOP/s")
                    if bwd:
                        line += f"  bwd {r['bwd_ms']:.3f} ms {r['bwd_tflops']:.1f} TFLOP/s"
                    print(line, flush=True)
    for i in range(args.rounds):
        for name in (("SD1", "SD2_BASE") if i % 2 == 0 else ("SD2_BASE", "SD1")):
            r = unet_passes(name, args.iters)
            result["unet"].append(r)
            print(f"unet {name}: forward b{SAMPLE_B} {r['unet_fwd_b16_ms']:.2f} ms  forward+backward b{TRAIN_B} "
                  f"{r['unet_fwd_bwd_b40_ms']:.1f} ms  peak {r['peak_gib']:.1f} GiB", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
