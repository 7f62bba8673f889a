"""ncu / timing target (not a test): GroupNorm forward (finalize + apply), GroupNorm backward and LayerNorm at the
U-Net's dominant shapes.
    python tests/prof_norm.py                       # CUDA-event timings -> achieved GB/s on ALGORITHMIC bytes
    ncu --set full --clock-control none --import-source on -k regex:"gn_|layernorm" -c 24 -o gpurun_out/r2_norm_full \
        python tests/prof_norm.py --once
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddpo_b200 import ops  # noqa: E402

dev = "cuda"
once = "--once" in sys.argv
g = torch.Generator(device="cpu").manual_seed(0)
PEAK = 6576.4


def slab_stats(x2d):
    t = x2d.view(-1, 32, x2d.shape[1]).double()
    return torch.stack([t.sum(1), (t * t).sum(1)], -1).float().contiguous()


def timeit(fn, reps):
    # inputs are 80+ MB each: larger than what stays in L2 between calls of different tensors; alternate two input sets
    for _ in range(0 if once else 3):
        fn(0), fn(1)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(reps):
        fn(i & 1)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e-3


def gn_fwd(b, hw, c0, c1, with_stats=True, tag=""):
    c = c0 + c1
    sets = []
    for _ in range(2):
        x0 = torch.randn(b, hw, c0, generator=g).to(dev)
        x1 = torch.randn(b, hw, c1, generator=g).to(dev) if c1 else None
        s0 = slab_stats(x0.view(b * hw, c0)) if with_stats else None
        s1 = slab_stats(x1.view(b * hw, c1)) if (c1 and with_stats) else None
        sets.append((x0, x1, s0, s1))
    sc, bi = torch.ones(c, device=dev), torch.zeros(c, device=dev)
    ws = torch.zeros(ops.groupnorm_workspace_floats(b, hw, c), device=dev)
    y = torch.zeros(b, hw, c, dtype=torch.bfloat16, device=dev)

    def run(i):
        x0, x1, s0, s1 = sets[i]
        ops.groupnorm_fwd(x0, sc, bi, ws, b, hw, c0, x1=x1, c1=c1, silu=True, y_bf16=y, stats0=s0, stats1=s1)

    def run_stats_only(i):
        x0, x1, s0, s1 = sets[i]
        ops.groupnorm_fwd(x0, sc, bi, ws, b, hw, c0, x1=x1, c1=c1, silu=True, stats0=s0, stats1=s1)

    def run_apply_only(i):
        x0, x1, s0, s1 = sets[i]
        ops.groupnorm_fwd(x0, sc, bi, ws, b, hw, c0, x1=x1, c1=c1, silu=True, y_bf16=y, skip_stats=True)
    t = timeit(run, 1 if once else 20)
    alg = b * hw * c * 6
    line = (f"gn_fwd{tag} B{b} hw{hw} C{c0}+{c1} stats={with_stats}: {t * 1e6:8.1f} us  {alg / t / 1e9:7.0f} GB/s algorithmic "
            f"({alg / t / 1e9 / PEAK:.2f} of {PEAK:.0f})")
    if not once:
        ts, ta = timeit(run_stats_only, 20), timeit(run_apply_only, 20)
        line += f" | statistics alone {ts * 1e6:6.1f} us, apply alone {ta * 1e6:6.1f} us ({alg / ta / 1e9:5.0f} GB/s)"
    print(line, flush=True)


def gn_bwd(b, hw, c):
    sets = []
    for _ in range(2):
        sets.append((torch.randn(b, hw, c, generator=g).to(dev), torch.randn(b, hw, c, generator=g).to(dev)))
    sc, bi = torch.ones(c, device=dev), torch.zeros(c, device=dev)
    ws = torch.zeros(ops.groupnorm_workspace_floats(b, hw, c), device=dev)
    y = torch.zeros(b, hw, c, dtype=torch.bfloat16, device=dev)
    dx = torch.zeros(b, hw, c, device=dev)
    dsc, dbi = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
    ops.groupnorm_fwd(sets[0][0], sc, bi, ws, b, hw, c, silu=True, y_bf16=y)

    def run(i):
        x, dy = sets[i]
        ops.groupnorm_bwd(x, sc, bi, ws, b, hw, c, dy, dx, dsc, dbi, silu=True, accumulate=False)
    t = timeit(run, 1 if once else 10)
    alg = b * hw * c * 12
    print(f"gn_bwd B{b} hw{hw} C{c}: {t * 1e6:8.1f} us  {alg / t / 1e9:7.0f} GB/s algorithmic ({alg / t / 1e9 / PEAK:.2f})")


def ln_fwd(m, c):
    xs = [torch.randn(m, c, generator=g).to(dev) for _ in range(2)]
    sc, bi = torch.ones(c, device=dev), torch.zeros(c, device=dev)
    y = torch.zeros(m, c, dtype=torch.bfloat16, device=dev)
    st = torch.zeros(m, 2, device=dev)
    t = timeit(lambda i: ops.layernorm_fwd(xs[i], sc, bi, y, m, c, stats=st), 1 if once else 20)
    alg = m * c * 6
    print(f"ln_fwd M{m} C{c}: {t * 1e6:8.1f} us  {alg / t / 1e9:7.0f} GB/s algorithmic ({alg / t / 1e9 / PEAK:.2f})")


def ln_bwd(m, c):
    xs = [(torch.randn(m, c, generator=g).to(dev), torch.randn(m, c, generator=g).to(dev)) for _ in range(2)]
    sc, bi = torch.ones(c, device=dev), torch.zeros(c, device=dev)
    y = torch.zeros(m, c, dtype=torch.bfloat16, device=dev)
    st = torch.zeros(m, 2, device=dev)
    ops.layernorm_fwd(xs[0][0], sc, bi, y, m, c, stats=st)
    dx = torch.zeros(m, c, device=dev)
    dsc, dbi = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
    ws = torch.zeros(ops.layernorm_bwd_workspace_floats(m, c), device=dev)
    t = timeit(lambda i: ops.layernorm_bwd(xs[i][0], sc, st, xs[i][1], dx, dsc, dbi, ws, m, c, accumulate=True), 1 if once else 10)
    alg = m * c * 16
    print(f"ln_bwd M{m} C{c}: {t * 1e6:8.1f} us  {alg / t / 1e9:7.0f} GB/s algorithmic ({alg / t / 1e9 / PEAK:.2f})")


gn_fwd(16, 4096, 320, 0)            # the dominant sampling shape
gn_fwd(16, 4096, 320, 0, with_stats=False, tag="[two-pass]")
gn_fwd(16, 4096, 640, 320)          # up_blocks_3 concat
gn_fwd(16, 1024, 640, 0)
gn_fwd(16, 256, 1280, 1280)
gn_fwd(40, 4096, 320, 0)            # training batch
ln_fwd(65536, 320)
ln_fwd(16384, 640)
ln_fwd(4096, 1280)
if not once:
    gn_bwd(40, 4096, 320)
    gn_bwd(40, 1024, 640)
    ln_bwd(163840, 320)
    ln_bwd(40960, 640)
print("done")
