"""ncu target (not a test): weight-gradient GEMMs of the level-0 (320-channel, 64x64) layers at training batch 40.
    ncu --set full --clock-control none --import-source on -k regex:wgrad -o gpurun_out/prof_wgrad python tests/prof_wgrad.py
"""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddpo_b200 import ops

dev = "cuda"
g = torch.Generator(device="cpu").manual_seed(0)
B = int(os.environ.get("PROF_B", 40))
x = torch.randn(B, 64, 64, 320, generator=g).to(dev).to(torch.bfloat16)
dy = torch.randn(B * 4096, 320, generator=g).to(dev).to(torch.bfloat16)
dw9 = torch.zeros(2880, 320, device=dev)
dw1 = torch.zeros(320, 320, device=dev)
x2 = torch.randn(B, 16, 16, 1280, generator=g).to(dev).to(torch.bfloat16)
dy2 = torch.randn(B * 256, 1280, generator=g).to(dev).to(torch.bfloat16)
dw2 = torch.zeros(11520, 1280, device=dev)


def t(fn, n=10):
    for _ in range(2): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


a = t(lambda: ops.wgrad(dy=dy, n=320, x0=x, c0=320, conv=(B, 64, 64), taps=9, dw=dw9))
b = t(lambda: ops.wgrad(dy=dy, n=320, x0=x, c0=320, m=B * 4096, dw=dw1))
c = t(lambda: ops.wgrad(dy=dy2, n=1280, x0=x2, c0=1280, conv=(B, 16, 16), taps=9, dw=dw2))
print(f"conv3x3 320->320 {a:.1f} us ({2 * B * 4096 * 2880 * 320 / a / 1e6:.0f} TF/s) | linear 320x320 {b:.1f} us | "
      f"conv3x3 1280->1280 @16x16 {c:.1f} us ({2 * B * 256 * 11520 * 1280 / c / 1e6:.0f} TF/s)")
