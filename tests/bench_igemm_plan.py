"""Micro-benchmark (not a test): every distinct implicit-GEMM launch of one SD2-base denoising step (batch 16) and one
PPO train pass (batch 40), timed with CUDA events under the planned tile and under the tile the library used before
(128 rows, width from N alone), alternating in one process.  ``--all`` also times every other tile of each launch.

    python tests/bench_igemm_plan.py [--all] [--rounds R] [--iters I] [--json PATH]
"""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import _igemm_census as ic  # noqa: E402
from _forward_census import Tensor  # noqa: E402
from ddpo_b200 import _lib, ops  # noqa: E402

DEV = "cuda"


def materialize(t, g):
    """a tensor of the recorded shape, dtype and strides, on a buffer of its own"""
    numel = 1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride))
    base = torch.randn(numel, generator=g, device=DEV).to(t.dtype) if t.dtype.is_floating_point else \
        torch.zeros(numel, dtype=t.dtype, device=DEV)
    return base.as_strided(t.shape, t.stride)


def time_tiles(call, tiles, rounds, iters):
    """{tile: median ms per launch over alternating rounds}"""
    g = torch.Generator(device=DEV).manual_seed(0)
    kw = {k: materialize(v, g) if isinstance(v, Tensor) else v for k, v in call.args.items()}
    kw.pop("bm", None), kw.pop("bn", None)
    runs = {t: [] for t in tiles}
    for t in tiles:
        for _ in range(3):
            ops.igemm(**kw, bm=t[0], bn=t[1])
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(rounds):
        for t in tiles:
            ev[0].record()
            for _ in range(iters):
                ops.igemm(**kw, bm=t[0], bn=t[1])
            ev[1].record()
            torch.cuda.synchronize()
            runs[t].append(ev[0].elapsed_time(ev[1]) / iters)
    return {t: sorted(v)[len(v) // 2] for t, v in runs.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--all", action="store_true", help="also time every other tile that fits each launch")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_igemm_plan.py needs a CUDA device"
    name = torch.cuda.get_device_name(0)
    print(f"# {name}", flush=True)
    report = {"device": name, "passes": {}}
    for pass_name in ("sample", "train"):
        rows, tot_new, tot_old, tot_flop = [], 0.0, 0.0, 0.0
        for call, count in ic.distinct(pass_name):
            m, n, k, geglu = ic.shape(call)
            new = ops.igemm_plan(m, n, k, geglu)[:2]
            old = (128, ic.old_width(n, geglu))
            tiles = [new] if new == old else [new, old]
            if args.all:
                for bm in (64, 128):
                    for bn in (32, 64, 96, 128, 160, 192, 256):
                        if (bm, bn) in tiles or n % bn or (geglu and bn != old[1]):
                            continue
                        try:
                            ops.igemm_plan(m, n, k, geglu, bm=bm, bn=bn)
                        except _lib.DdpoError:
                            continue
                        tiles.append((bm, bn))
            ms = time_tiles(call, tiles, args.rounds, args.iters)
            flop = 2.0 * m * n * k
            tot_new += count * ms[new]
            tot_old += count * ms[old]
            tot_flop += count * flop
            rows.append(dict(sig=call.tag(), count=count, m=m, n=n, k=k, geglu=geglu, plan=list(new), old=list(old),
                             ms={f"{t[0]}x{t[1]}": v for t, v in ms.items()}))
            print(f"{pass_name:6s} x{count:<3d} {call.tag():60s} plan {new[0]:3d}x{new[1]:<3d} "
                  f"{flop / ms[new] / 1e9:6.1f} TF/s  old {old[0]}x{old[1]:<3d} {flop / ms[old] / 1e9:6.1f} TF/s  "
                  f"{ms[old] / ms[new]:5.3f}x", flush=True)
        summary = dict(ms_new=tot_new, ms_old=tot_old, tflops_new=tot_flop / tot_new / 1e9,
                       tflops_old=tot_flop / tot_old / 1e9)
        report["passes"][pass_name] = dict(summary, launches=rows)
        print(f"# {pass_name}: igemm total {tot_new:.2f} ms planned ({summary['tflops_new']:.1f} TF/s) vs "
              f"{tot_old:.2f} ms before ({summary['tflops_old']:.1f} TF/s)", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
