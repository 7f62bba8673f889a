"""ncu target (not a test): the kernels around the U-Net -- one VAE decode of 2 latents at SD size, one CLIP text
encode of 8 prompts (SD2 tower), the RWR input/loss kernels and the trajectory gather -- bracketed by
cudaProfilerStart/Stop after a warm-up pass.

    ncu --profile-from-start off --csv --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum \
        python tests/prof_aux.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddpo_b200 import ops  # noqa: E402
from ddpo_b200.text_encoder import SD2_TEXT, CLIPTextEncoder  # noqa: E402
from ddpo_b200.vae import SD_VAE, VAEDecoder  # noqa: E402

dev = "cuda"
g = torch.Generator().manual_seed(0)
dec = VAEDecoder(SD_VAE, device=dev, seed=0, decode_batch=2)
enc = CLIPTextEncoder(SD2_TEXT, device=dev, seed=1)
lat = (torch.randn(2, 4, 64, 64, generator=g) * 0.18215).to(dev)
ids = torch.randint(3, 49408, (8, 77), generator=g).numpy()
mom = torch.randn(8, 64, 64, 8, generator=g).to(dev)
keys = ops.key_tensor([(1, 2), (3, 4)], dev)
ts = torch.randint(0, 1000, (8,), generator=g).to(dev, torch.int32)
ac = torch.linspace(0.999, 0.005, 1000).to(dev)
noise, noisy = torch.empty(8, 4, 64, 64, device=dev), torch.empty(8, 4, 64, 64, device=dev)
eps = torch.randn(16, 16384, generator=g).to(dev)
d_eps = torch.empty_like(eps)
loss, ws = torch.zeros(1, device=dev), ops.rwr_workspace(8, dev)
traj = torch.randn(8 * 51, 16384, generator=g).to(dev)
idx = torch.randint(0, 8 * 51, (20,), generator=g).to(dev)
dst = torch.empty(20, 16384, device=dev)


def once():
    dec.decode(lat)
    enc(ids)
    ops.rwr_noisy_latents(mom, keys[0], keys[1], ts, ac, noise, noisy)
    ops.rwr_mse_loss(eps[:8], eps[8:], noise.view(8, -1), 5.0, loss, ws, d_eps_u=d_eps[:8], d_eps_c=d_eps[8:])
    ops.gather_rows(traj, idx, dst)


once()
torch.cuda.synchronize()
torch.cuda.profiler.start()
once()
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("done")
