"""Micro-benchmark (not a test): every distinct weight-gradient GEMM of one SD2-base PPO train pass (batch 40), timed
with CUDA events, with the plan it runs and its rate.  Run it from two trees (e.g. before and after a planner change)
in one GPU session to compare them; a build without ``wgrad_plan`` prints the plan its own rules give.

``--all`` also times, per call, every other width that divides N at the planned split count, and the planned width at
one split and at the split count of the previous planner.  ``--accuracy`` measures, per call, the relative L2 error
against float64 of the planned split count and of the previous planner's (same width, seeded Gaussian operands).

    python tests/bench_wgrad_plan.py [--cfg sd2] [--all] [--accuracy] [--rounds R] [--iters I] [--json PATH]
"""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import _wgrad_census as wc  # noqa: E402
from _forward_census import Tensor  # noqa: E402
from bench_igemm_plan import materialize  # noqa: E402
from ddpo_b200 import ops  # noqa: E402

DEV = "cuda"


def operands(call):
    g = torch.Generator(device=DEV).manual_seed(0)
    return {k: materialize(v, g) if isinstance(v, Tensor) else v for k, v in call.args.items()}


def time_call(kw, rounds, iters, **plan):
    """median ms per call over ``rounds`` windows of ``iters`` calls"""
    for _ in range(3):
        ops.wgrad(**kw, **plan)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    runs = []
    for _ in range(rounds):
        ev[0].record()
        for _ in range(iters):
            ops.wgrad(**kw, **plan)
        ev[1].record()
        torch.cuda.synchronize()
        runs.append(ev[0].elapsed_time(ev[1]) / iters)
    return sorted(runs)[len(runs) // 2]


def rel_error(kw, **plan):
    """relative L2 error against float64 of dW computed from zero"""
    from test_param_grad_layers import _wgrad_ref
    rows2d = lambda t: t if t.dim() == 2 else t.reshape(-1, t.shape[-1])   # noqa: E731
    assert kw.get("x1") is None
    x, dy = rows2d(kw["x0"])[:, :kw["c0"]], rows2d(kw["dy"])[:, :kw["n"]]
    ref, _ = _wgrad_ref(x, dy, kw.get("conv"), kw.get("taps", 1), kw.get("stride", 1))
    dw = kw["dw"]
    dw.zero_()
    ops.wgrad(**kw, **plan)
    err = ((dw.double().reshape(ref.shape) - ref).norm() / ref.norm()).item()
    del ref
    return err


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", default="sd2", choices=sorted(wc.CONFIGS))
    ap.add_argument("--all", action="store_true", help="also time other widths and split counts of each call")
    ap.add_argument("--accuracy", action="store_true", help="error against float64, planned vs previous split count")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_wgrad_plan.py needs a CUDA device"
    name = torch.cuda.get_device_name(0)
    print(f"# {name}", flush=True)
    planner = hasattr(ops, "wgrad_plan")
    rows, tot_ms, tot_flop = [], 0.0, 0.0
    err_sq = {"planned": 0.0, "previous": 0.0}
    for call, count in wc.distinct(args.cfg):
        m, c0, c1, n, taps = wc.shape(call)
        old_s = wc.old_plan(m, c0, c1, n, taps)[0]
        kw = operands(call)
        if planner:
            bn, splits = ops.wgrad_plan(m, c0, n, c1, taps)
            plan = f"{bn}x{splits}"
        else:
            plan = f"old {old_s} splits, CTAs {wc.old_plan(m, c0, c1, n, taps)[1]}"
        ms = time_call(kw, args.rounds, args.iters)
        flop = 2.0 * m * n * taps * (c0 + c1)
        tot_ms += count * ms
        tot_flop += count * flop
        row = dict(sig=call.tag(), count=count, m=m, c0=c0, c1=c1, n=n, taps=taps, plan=plan, ms=ms)
        line = f"x{count:<3d} {call.tag():70s} {plan:28s} {ms * 1e3:8.1f} us {flop / ms / 1e9:6.1f} TF/s"
        if planner and args.all:
            others = [(w, splits) for w in (64, 128, 192, 256, 320) if n % w == 0 and w != bn]
            others += [(bn, s) for s in {1, old_s} if s != splits]
            row["others"] = {f"{w}x{s}": time_call(kw, args.rounds, args.iters, bn=w, splits=s) for w, s in others}
            line += "  | " + " ".join(f"{k} {flop / v / 1e9:5.0f}" for k, v in row["others"].items())
        if planner and args.accuracy:
            row["err"] = {"planned": rel_error(kw), "previous": rel_error(kw, bn=bn, splits=old_s)}
            for k, v in row["err"].items():
                err_sq[k] += count * v * v
            line += f"  | rel err planned {row['err']['planned']:.2e} ({splits} splits), " \
                    f"previous {row['err']['previous']:.2e} ({old_s})"
        rows.append(row)
        print(line, flush=True)
        del kw
    print(f"# wgrad total {tot_ms:.2f} ms per pass ({tot_flop / tot_ms / 1e9:.1f} TF/s)", flush=True)
    if planner and args.accuracy:
        k = len(wc.calls(args.cfg))
        print(f"# rms relative error over the pass's calls: planned {(err_sq['planned'] / k) ** 0.5:.3e}, "
              f"previous split counts {(err_sq['previous'] / k) ** 0.5:.3e}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(device=name, cfg=args.cfg, ms=tot_ms, tflops=tot_flop / tot_ms / 1e9, calls=rows), f, indent=1)


if __name__ == "__main__":
    main()
