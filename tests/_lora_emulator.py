"""TEST INFRASTRUCTURE: the CPU ops emulator (tests/_cpu_ops_emulator.py) plus torch-CPU emulations of the two LoRA
entry points, ``ops.lora_merge`` and ``ops.lora_grad``, with the same argument conventions.  The host-side dry runs of
the LoRA mode patch this module in as ``ops``; the product never imports it."""
import torch

from _cpu_ops_emulator import *  # noqa: F401,F403
from _cpu_ops_emulator import BF16

LORA_RANKS = (4, 8, 16)


def lora_merge(w, down, up, k, n, rank, fwd=None, ldk=0, row_offset=0, dgrad=None, ld_dst=0, col_offset=0, merged=None,
               scale=1.0):
    v = w.reshape(k, n) + scale * (down.reshape(k, rank) @ up.reshape(rank, n))
    if fwd is not None:
        fwd.reshape(-1, ldk or k)[row_offset:row_offset + n, :k] = v.t().to(BF16)
    if dgrad is not None:
        dgrad.reshape(k, ld_dst or n)[:, col_offset:col_offset + n] = v.to(BF16)
    if merged is not None:
        merged.copy_(v.reshape(merged.shape))


def lora_grad(x, dys, downs, ups, d_downs, d_ups, m, k, n, rank, ldx=0, lddy=0, scale=1.0):
    xf = x.reshape(m, -1)[:, :k].float()
    for dy, d, u, dd, du in zip(dys, downs, ups, d_downs, d_ups):
        # a column slice of a wider [m, lddy] buffer: rebuild the [m, n] view from the flat storage
        dyf = dy.as_strided((m, n), (lddy or n, 1)).float()
        du += scale * ((xf @ d).t() @ dyf)
        dd += scale * (xf.t() @ (dyf @ u.t()))
