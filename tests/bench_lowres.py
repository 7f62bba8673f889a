"""Micro-benchmark (not a test): low-resolution convolutions (few CTA tiles) across tile widths BN."""
import os, sys, math
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddpo_b200 import ops
dev = "cuda"
g = torch.Generator(device="cpu").manual_seed(0)

def timeit(fn, iters=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3

for (b, h, c, n) in [(40, 8, 1280, 1280), (16, 8, 1280, 1280), (40, 16, 1280, 1280), (16, 16, 1280, 1280)]:
    a = torch.randn(b, h, h, c, generator=g).to(dev).to(torch.bfloat16)
    w = torch.randn(n, 9 * c, generator=g).to(dev).to(torch.bfloat16)
    out = torch.zeros(b * h * h, n, device=dev)
    line = [f"conv {b}x{h}x{h} c{c}->{n}"]
    for bn in (0, 256, 160, 128, 64):
        t = timeit(lambda: ops.igemm(a0=a, wt=w, n=n, c0=c, conv=(b, h, h), taps=9, out_f32=out, bn=bn))
        line.append(f"bn{bn} {t:6.1f}us")
    print(" | ".join(line), flush=True)
