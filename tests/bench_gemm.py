"""Micro-benchmark (not a test): igemm with fp32 and bf16 outputs on a few representative shapes. Usage: python tests/bench_gemm.py"""
import math, os, sys, time
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
    return e0.elapsed_time(e1) / iters * 1e-3

def run(name, m=None, k=None, n=None, conv=None, c=None, taps=9, bn=0, res=False):
    if conv is None:
        a = torch.randn(m, k, generator=g).to(dev).to(torch.bfloat16)
        w = torch.randn(n, k, generator=g).to(dev).to(torch.bfloat16)
        flops = 2.0 * m * n * k
    else:
        b, h = conv
        a = torch.randn(b, h, h, c, generator=g).to(dev).to(torch.bfloat16)
        w = torch.randn(n, taps * c, generator=g).to(dev).to(torch.bfloat16)
        m = b * h * h
        flops = 2.0 * m * n * taps * c
    out = torch.zeros(m, n, device=dev)
    outb = torch.zeros(m, n, dtype=torch.bfloat16, device=dev)
    r = torch.randn(m, n, device=dev) if res else None
    line = [name]
    for outk in ("f32", "bf16"):
        def fn():
            if conv is None:
                ops.igemm(a0=a, wt=w, n=n, c0=k, m=m, residual=r, out_f32=out if outk == "f32" else None,
                          out_bf16=outb if outk == "bf16" else None, bn=bn)
            else:
                ops.igemm(a0=a, wt=w, n=n, c0=c, conv=(conv[0], conv[1], conv[1]), taps=taps, residual=r,
                          out_f32=out if outk == "f32" else None, out_bf16=outb if outk == "bf16" else None, bn=bn)
        t = timeit(fn)
        line.append(f"{outk}: {flops / t / 1e12:7.1f} TF/s ({t * 1e6:7.1f} us)")
    print(" | ".join(line), flush=True)

run("linear 16384x1280x8192 bn256", m=16384, k=8192, n=1280)
run("linear 16384x1280x8192 bn128", m=16384, k=8192, n=1280, bn=128)
run("linear 65536x320x2880 bn160", m=65536, k=2880, n=320)
run("linear 65536x320x320", m=65536, k=320, n=320, res=True)
run("linear 65536x2560x320", m=65536, k=320, n=2560)
run("conv 16x64x64 c320->320", conv=(16, 64), c=320, n=320, res=True)
run("conv 16x64x64 c640->640", conv=(16, 64), c=640, n=640)
run("conv 16x16x16 c1280->1280", conv=(16, 16), c=1280, n=1280)
run("conv 16x8x8 c1280->1280", conv=(16, 8), c=1280, n=1280)
run("conv1x1 16x64x64 c960->320", conv=(16, 64), c=960, n=320, taps=1)
